// abi_many_krylov.cuh -- amgb_solve_many_cg / amgb_solve_many_bicgstab: MultilevelSolver.solve_many(accel='cg' |
// 'bicgstab'), the GPU-resident CG and BiCGStab of abi_krylov.cuh on up to eight right-hand sides per pass over the
// hierarchy (included by engine.cu after abi_many.cuh).
//
// Each group driver is a line-by-line K-wide restatement of amgb_solve_cg / amgb_solve_bicgstab: the preconditioner
// is the batched cycle from zero (many_one_iteration), the SpMVs and residuals are many_spmv on the level-0 operator,
// the dot products are many_dot_kernel + many_reduce_kernel (dev_dot's grid and order per column) and the vector
// updates many_axpby_kernel (axpby_kernel's expression per column).  So column j of the result -- iterate, residual
// list and info -- is what the single driver computes on column j, bit for bit.
//
// The scalars and the branch order of every column live on the host: status, residual list, and the aborts / stops
// in the single driver's order.  A column that stops leaves the active mask; many_axpby_kernel never writes an
// inactive column, so its iterate stays exactly the one it stopped with and all columns are unpacked at the end.
// Padding columns (groups of width 3, 5, 6, 7) are inactive from the start, so no 0/0 is formed for them.  Whole-block
// SpMVs, residuals and copies still touch inactive columns; columns never mix, so that changes no active column.
// The host reads K values per reduction; reads the single driver performs separately (r'z and ||r||^2) share one
// device-to-host copy, which changes no value.
#pragma once

enum { kManyCg = 0, kManyBicgstab = 1 };

template <int K>
struct ManyKrylov {
    amgb_hierarchy *h;
    ManyWidth &mw;
    ManyLevel &V;
    const DevCsr &A0;
    long long n;
    int cycle;
    bool dev;                    // the caller's blocks are device memory (AMGB_FLAG_DEVICE_IO)
    cudaStream_t s;
    std::vector<double> got;     // slot * K + q: the last values read

    ManyKrylov(amgb_hierarchy *h_, int cyc, bool dev_)
        : h(h_), mw(h_->many[many_index(K)]), V(mw.lv[0]), A0(h_->levels[0].A), n(h_->levels[0].A.n_rows), cycle(cyc),
          dev(dev_), s(h_->stream), got((size_t)2 * K) {}

    // <x_q, y_q> of the K columns -> norms2[slot*K ..) (dev_dot without the read)
    int dot(const double *x, const double *y, int slot)
    {
        many_dot_kernel<K><<<sumsq_blocks(h->S), 256, 0, s>>>(x, y, n, mw.partials);
        CK(cudaGetLastError());
        many_reduce_kernel<K><<<1, 1024, 0, s>>>(mw.partials, sumsq_blocks(h->S), mw.norms2 + (size_t)slot * K);
        CK(cudaGetLastError());
        h->launches += 2;
        return AMGB_OK;
    }
    int read(int slots)
    {
        CK(cudaMemcpyAsync(got.data(), mw.norms2, sizeof(double) * (size_t)slots * K, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return AMGB_OK;
    }
    // y_q = a[q] x_q + b[q] y_q on the columns in `active` (dev_axpby per column)
    int axpby(const double *a, const double *x, const double *b, double *y, unsigned active)
    {
        if (active == 0 || n <= 0) return AMGB_OK;
        ManyAxpby c = {};
        for (int q = 0; q < K; q++) { c.a[q] = a[q]; c.b[q] = b[q]; }
        c.active = active;
        many_axpby_kernel<K><<<vec_grid(h->S, n), 256, 0, s>>>(c, x, y, n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    }
    int copy(double *dst, const double *src)
    {
        CK(cudaMemcpyAsync(dst, src, sizeof(double) * (size_t)n * K, cudaMemcpyDeviceToDevice, s));
        return AMGB_OK;
    }
    int precond()                // V.x <- M V.b: one batched cycle from zero
    {
        V.x = V.x_home;
        RET(h->launch_count_fill(V.x, n * K));
        return many_one_iteration<K>(h, cycle, 1);
    }
    // columns [c0, c0+w) of the caller's n x k block -> dst (level-0 numbering, zero-padded); a host block is
    // staged through mw.io, a device block packed in place
    int load(const double *src, int32_t k, int c0, int w, double *dst)
    {
        if (dev) return many_load<K>(h, src + c0, k, w, dst);
        const size_t wb = sizeof(double) * (size_t)w;
        CK(many_copy_2d(mw.io, wb, src + c0, sizeof(double) * (size_t)k, wb, (size_t)n, cudaMemcpyHostToDevice, s));
        return many_load<K>(h, mw.io, w, w, dst);
    }
    int store(const double *src, int32_t k, int c0, int w, double *dst)
    {
        if (dev) return many_store<K>(h, src, 0, w, dst + c0, k);
        const size_t wb = sizeof(double) * (size_t)w;
        RET(many_store<K>(h, src, 0, w, mw.io, w));
        CK(many_copy_2d(dst + c0, sizeof(double) * (size_t)k, mw.io, wb, wb, (size_t)n, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return AMGB_OK;
    }
};

// K-wide level vectors (many_prepare) plus the first `nbuf` Krylov blocks of this width
template <int K>
static int many_krylov_prepare(amgb_hierarchy *h, int nbuf)
{
    RET(many_prepare<K>(h, 2));
    ManyWidth &mw = h->many[many_index(K)];
    const long long n = h->levels[0].A.n_rows;
    for (int i = 0; i < nbuf; i++)
        if (mw.kry[i] == nullptr) RET(h->dalloc(&mw.kry[i], n * K + 2));
    return AMGB_OK;
}

static void many_krylov_out(int32_t k, int c0, int w, const std::vector<std::vector<double>> &res,
                            const std::vector<int> &status, double *residuals, int32_t *n_residuals, int32_t *info)
{
    for (int q = 0; q < w; q++) {
        if (residuals != nullptr)
            for (size_t t = 0; t < res[(size_t)q].size(); t++) residuals[t * (size_t)k + c0 + q] = res[(size_t)q][t];
        if (n_residuals != nullptr) n_residuals[c0 + q] = (int32_t)res[(size_t)q].size();
        if (info != nullptr) info[c0 + q] = status[(size_t)q];
    }
}

// amgb_solve_cg on columns [c0, c0+w) of the caller's n x k blocks
template <int K>
static int many_cg_group(amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X, bool x0_zero,
                         bool dev,
                         double tol, int32_t maxiter, int32_t cycle, double *residuals, int32_t *n_residuals,
                         int32_t *info)
{
    RET(many_krylov_prepare<K>(h, 4));
    ManyKrylov<K> M(h, cycle, dev);
    ManyWidth &mw = M.mw;
    double *xk = mw.kry[0], *p = mw.kry[1], *Ap = mw.kry[2], *bk = mw.kry[3];
    double *r = M.V.b;                                    // CG residual = rhs of the preconditioner
    const double *z = M.V.x_home;                         // the preconditioner's output (many_cycle brings it home)
    RET(M.load(B, k, c0, w, bk));
    if (x0_zero) RET(h->launch_count_fill(xk, M.n * K));
    else RET(M.load(X, k, c0, w, xk));
    std::vector<double> normb((size_t)K, 1.0), rtol((size_t)K, 0.0), rz((size_t)K, 0.0), rz_old((size_t)K, 0.0);
    std::vector<double> alpha((size_t)K, 0.0), neg_alpha((size_t)K, 0.0), beta((size_t)K, 0.0), ones((size_t)K, 1.0);
    std::vector<std::vector<double>> res((size_t)w);
    std::vector<int> status((size_t)w, -2);
    unsigned act = 0;
    RET(M.dot(bk, bk, 0));
    RET(M.read(1));
    for (int q = 0; q < w; q++) {
        normb[(size_t)q] = std::sqrt(M.got[(size_t)q]);
        if (normb[(size_t)q] == 0.0) normb[(size_t)q] = 1.0;
    }
    RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));     // r = b - A x        (_cg.py:99)
    RET(M.precond());                                     // z = M r            (:100)
    RET(M.copy(p, z));                                    // p = z              (:101)
    RET(M.dot(r, z, 0));                                  // rz = <r, z>        (:102)
    RET(M.dot(r, r, 1));
    RET(M.read(2));
    for (int q = 0; q < w; q++) {
        rz[(size_t)q] = M.got[(size_t)q];
        res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));   // :104-106
        rtol[(size_t)q] = tol * normb[(size_t)q];                    // criteria 'rr' (:114-115)
        if (res[(size_t)q].back() < rtol[(size_t)q]) status[(size_t)q] = 0;   // :133-134
        else act |= 1u << q;
    }
    int it = 0;
    while (act != 0) {
        RET(many_spmv<K>(h, OP_SPMV, M.A0, p, nullptr, Ap));       // Ap = A p           (:142)
        rz_old = rz;
        RET(M.dot(Ap, p, 0));                                      // curvature of A     (:145-148)
        RET(M.read(1));
        for (int q = 0; q < w; q++) {
            if (!(act & (1u << q))) continue;
            const double pAp = M.got[(size_t)q];
            if (pAp < 0.0) { status[(size_t)q] = -1; act &= ~(1u << q); continue; }
            alpha[(size_t)q] = rz[(size_t)q] / pAp;                // :150
            neg_alpha[(size_t)q] = -alpha[(size_t)q];
        }
        if (act == 0) break;
        RET(M.axpby(alpha.data(), p, ones.data(), xk, act));       // x += alpha p       (:151)
        if ((it % 8) != 0 && it > 0) {
            RET(M.axpby(neg_alpha.data(), Ap, ones.data(), r, act));   // r -= alpha Ap  (:153-154)
        } else {
            RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));       // r = b - A x        (:155-156)
        }
        RET(M.precond());                                          // z = M r            (:158)
        RET(M.dot(r, z, 0));                                       // :159
        RET(M.dot(r, r, 1));                                       // (read with rz: r does not change before :171)
        RET(M.read(2));
        for (int q = 0; q < w; q++) {
            if (!(act & (1u << q))) continue;
            rz[(size_t)q] = M.got[(size_t)q];
            if (rz[(size_t)q] < 0.0) { status[(size_t)q] = -1; act &= ~(1u << q); continue; }   // :161-163
            beta[(size_t)q] = rz[(size_t)q] / rz_old[(size_t)q];  // :165
        }
        if (act == 0) break;
        RET(M.axpby(ones.data(), z, beta.data(), p, act));         // p = beta p + z     (:166-167)
        it++;
        for (int q = 0; q < w; q++) {
            if (!(act & (1u << q))) continue;
            res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));   // :171-174
            if (res[(size_t)q].back() < rtol[(size_t)q]) { status[(size_t)q] = 0; act &= ~(1u << q); }   // :190-191
            else if (it == maxiter) { status[(size_t)q] = it; act &= ~(1u << q); }                       // :193-194
        }
    }
    RET(M.store(xk, k, c0, w, X));
    many_krylov_out(k, c0, w, res, status, residuals, n_residuals, info);
    return AMGB_OK;
}

// amgb_solve_bicgstab on columns [c0, c0+w) of the caller's n x k blocks
template <int K>
static int many_bicgstab_group(amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X, bool x0_zero,
                               bool dev,
                               double tol, int32_t maxiter, int32_t cycle, double *residuals, int32_t *n_residuals,
                               int32_t *info)
{
    RET(many_krylov_prepare<K>(h, 8));
    ManyKrylov<K> M(h, cycle, dev);
    ManyWidth &mw = M.mw;
    double *xk = mw.kry[0], *p = mw.kry[1], *AMp = mw.kry[2], *bk = mw.kry[3];
    double *r = mw.kry[4], *rstar = mw.kry[5], *sv = mw.kry[6], *AMs = mw.kry[7];
    const double *Mv = M.V.x_home;                        // the preconditioner's output
    RET(M.load(B, k, c0, w, bk));
    if (x0_zero) RET(h->launch_count_fill(xk, M.n * K));
    else RET(M.load(X, k, c0, w, xk));
    auto precond_of = [&](const double *v) -> int {       // V.x <- M v
        RET(M.copy(M.V.b, v));
        return M.precond();
    };
    std::vector<double> rtol((size_t)K, 0.0), rrstar_old((size_t)K, 0.0), alpha((size_t)K, 0.0);
    std::vector<double> neg_alpha((size_t)K, 0.0), omega((size_t)K, 0.0), neg_omega((size_t)K, 0.0);
    std::vector<double> beta((size_t)K, 0.0), ones((size_t)K, 1.0);
    std::vector<std::vector<double>> res((size_t)w);
    std::vector<int> status((size_t)w, -2);
    unsigned act = 0;
    RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));     // r = b - A x             (_bicgstab.py:96)
    RET(M.dot(r, r, 0));
    RET(M.dot(bk, bk, 1));
    RET(M.read(2));
    for (int q = 0; q < w; q++) {
        res[(size_t)q].push_back(std::sqrt(M.got[(size_t)q]));       // :97-100
        double normb = std::sqrt(M.got[(size_t)K + q]);
        if (normb == 0.0) normb = 1.0;                               // :103-106
        rtol[(size_t)q] = tol * normb;                               // criteria 'rr' (:109-110)
        if (res[(size_t)q].back() < rtol[(size_t)q]) status[(size_t)q] = 0;   // :122-123
        else act |= 1u << q;
    }
    if (act != 0) {
        RET(M.copy(rstar, r));                                       // :131-132
        RET(M.copy(p, r));
        RET(M.dot(rstar, r, 0));                                     // :134
        RET(M.read(1));
        for (int q = 0; q < w; q++) rrstar_old[(size_t)q] = M.got[(size_t)q];
    }
    int it = 0;
    while (act != 0) {
        RET(precond_of(p));                                          // Mp = M p                (:140)
        RET(many_spmv<K>(h, OP_SPMV, M.A0, Mv, nullptr, AMp));      // AMp = A Mp              (:141)
        RET(M.dot(rstar, AMp, 0));
        RET(M.read(1));
        for (int q = 0; q < w; q++) {
            alpha[(size_t)q] = (act & (1u << q)) ? rrstar_old[(size_t)q] / M.got[(size_t)q] : 0.0;   // :144
            neg_alpha[(size_t)q] = -alpha[(size_t)q];
        }
        RET(M.axpby(alpha.data(), Mv, ones.data(), xk, act));       // x += alpha Mp           (:155, first term)
        RET(M.copy(sv, r));
        RET(M.axpby(neg_alpha.data(), AMp, ones.data(), sv, act));  // s = r - alpha AMp       (:147)
        RET(precond_of(sv));                                         // Ms = M s                (:148)
        RET(many_spmv<K>(h, OP_SPMV, M.A0, Mv, nullptr, AMs));      // AMs = A Ms              (:149)
        RET(M.dot(AMs, sv, 0));
        RET(M.dot(AMs, AMs, 1));
        RET(M.read(2));
        for (int q = 0; q < w; q++) {
            omega[(size_t)q] = (act & (1u << q)) ? M.got[(size_t)q] / M.got[(size_t)K + q] : 0.0;   // :152
            neg_omega[(size_t)q] = -omega[(size_t)q];
        }
        RET(M.axpby(omega.data(), Mv, ones.data(), xk, act));       // x += omega Ms           (:155, second term)
        RET(M.copy(r, sv));
        RET(M.axpby(neg_omega.data(), AMs, ones.data(), r, act));   // r = s - omega AMs       (:158)
        RET(M.dot(rstar, r, 0));                                     // :161
        RET(M.dot(r, r, 1));                                         // (read with r*'r: r does not change before :170)
        RET(M.read(2));
        for (int q = 0; q < w; q++) {
            if (!(act & (1u << q))) continue;
            const double rrstar_new = M.got[(size_t)q];
            beta[(size_t)q] = (rrstar_new / rrstar_old[(size_t)q]) * (alpha[(size_t)q] / omega[(size_t)q]);   // :162
            rrstar_old[(size_t)q] = rrstar_new;
        }
        RET(M.axpby(neg_omega.data(), AMp, ones.data(), p, act));   // p - omega AMp
        RET(M.axpby(ones.data(), r, beta.data(), p, act));          // p = r + beta (p - omega AMp)   (:166)
        it++;
        for (int q = 0; q < w; q++) {
            if (!(act & (1u << q))) continue;
            res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));   // :170-173
            if (res[(size_t)q].back() < rtol[(size_t)q]) { status[(size_t)q] = 0; act &= ~(1u << q); }   // :184-185
            else if (it == maxiter) { status[(size_t)q] = it; act &= ~(1u << q); }                       // :187-188
        }
    }
    RET(M.store(xk, k, c0, w, X));
    many_krylov_out(k, c0, w, res, status, residuals, n_residuals, info);
    return AMGB_OK;
}

template <int K>
static int many_krylov_group(int method, amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X,
                             bool x0_zero, bool dev, double tol, int32_t maxiter, int32_t cycle, double *residuals,
                             int32_t *n_residuals, int32_t *info)
{
    if (method == kManyCg)
        return many_cg_group<K>(h, k, c0, w, B, X, x0_zero, dev, tol, maxiter, cycle, residuals, n_residuals, info);
    return many_bicgstab_group<K>(h, k, c0, w, B, X, x0_zero, dev, tol, maxiter, cycle, residuals, n_residuals, info);
}

static int many_krylov(int method, amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host, double tol,
                       int32_t maxiter, int32_t cycle, int32_t flags, double *residuals, int32_t *n_residuals,
                       int32_t *info)
{
    RET(check_many_args(h, k, cycle, 1, B_host, X_host));
    if (maxiter < 1) return fail(AMGB_EINVAL, "Number of iterations must be positive");
    if (method == kManyBicgstab && h->levels[0].A.n_rows < 2)
        return fail(AMGB_EINVAL, "bicgstab: n < 2 is the caller's closed form (b / A[0,0])");
    CallerIo io(h, flags);
    RET(io.begin(B_host, X_host));
    const bool x0_zero = (flags & AMGB_FLAG_X0_ZERO) != 0;
    h->launches = 0;
    for (int c0 = 0; c0 < k; c0 += 8) {
        const int w = std::min(8, k - c0);
        switch (many_width(w)) {
        case 2: RET(many_krylov_group<2>(method, h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                         residuals, n_residuals, info)); break;
        case 4: RET(many_krylov_group<4>(method, h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                         residuals, n_residuals, info)); break;
        default: RET(many_krylov_group<8>(method, h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                          residuals, n_residuals, info)); break;
        }
    }
    h->last_launches = h->launches;
    return io.end();
}

extern "C" int amgb_solve_many_cg(amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host, double tol,
                                  int32_t maxiter, int32_t cycle, int32_t flags, double *residuals,
                                  int32_t *n_residuals, int32_t *info)
{
    return many_krylov(kManyCg, h, k, B_host, X_host, tol, maxiter, cycle, flags, residuals, n_residuals, info);
}

extern "C" int amgb_solve_many_bicgstab(amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host,
                                        double tol, int32_t maxiter, int32_t cycle, int32_t flags, double *residuals,
                                        int32_t *n_residuals, int32_t *info)
{
    return many_krylov(kManyBicgstab, h, k, B_host, X_host, tol, maxiter, cycle, flags, residuals, n_residuals, info);
}
