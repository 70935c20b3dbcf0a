// abi_many_gmres.cuh -- amgb_solve_many_gmres: MultilevelSolver.solve_many(accel='gmres' | 'fgmres' | 'gmres_mgs'), the
// GPU-resident Householder, flexible and modified Gram-Schmidt GMRES of abi_krylov.cuh on up to eight right-hand sides
// per pass over the hierarchy (included by engine.cu after abi_many_krylov.cuh).
//
// many_gmres_group restates amgb_solve_gmres line by line on n x K blocks: the preconditioner is the batched cycle
// from zero, the level-0 SpMVs and residuals are many_spmv, the inner products many_dot_kernel / many_sumsq_from_kernel
// + many_reduce_kernel (dot_to's grid and order per column), and every vector kernel is the K-wide twin of the single
// driver's kernel (multi_rhs_kernels.cuh).  So column j -- iterate, residual list and info -- is what amgb_solve_gmres
// computes on column j, bit for bit.
//
// Numbering.  The reflectors single out leading rows, so the Krylov vectors stay in the original numbering; the
// gathers into and out of the level-0 numbering are many_pack_kernel with order0 / pos0 (a block copy when level 0
// is not permuted).
//
// Control flow.  Outer iterations run in step for all columns, and inside one every column still in the inner loop
// has the same `inner`, so the reflector loops are shared.  A column leaves the inner mask when its estimate meets
// the tolerance; its H, g and inner count are then final on the host and no kernel writes its reflectors again.  At
// the end of the outer iteration each column solves its own triangular system and forms its update (Horner scheme,
// or Z y for FGMRES) masked to the columns whose Krylov dimension exceeds the step; the update, the residual, the
// stagnation and stop tests follow per column.  A column with a status leaves every mask: its iterate is frozen and
// unpacked with the others at the end.  Padding columns and columns that meet the tolerance before the first
// iteration never enter a mask, so no 0/0 is formed for them.  Whole-block copies, SpMVs and cycles still touch
// inactive columns; columns never mix, so that changes no active column.
//
// Host state per column: H, the Givens rotations, g, y, niter, status and the residual list.  Per inner iteration
// the host reads the leading min(n, max_inner + 1) rows of v (m2 x K contiguous doubles) together with the K norms
// of v's tail in one copy, and K scalars for the new reflector's norm.
//
// Memory.  The reflector store is K x (max_inner + 1) x npad doubles (plus K x max_inner x npad of Z for FGMRES):
// one store per hierarchy, grown when a larger shape is asked.  Each call picks its width before computing: the
// widest the columns need, then narrower ones while the buffers do not fit; if even K = 2 does not fit the call
// returns AMGB_ENOTIMPL and the caller solves column by column.  Results do not depend on the width.
//
// Modified Gram-Schmidt (AMGB_FLAG_MGS, many_gmres_mgs_group) restates abi_krylov.cuh's gmres_mgs the same way, with
// one difference in layout: MGS needs no leading rows, so its basis, r and x stay in the level-0 numbering (no
// per-iteration gathers) and the store's W slots hold the Krylov basis, (max_inner + 1) x npad x K doubles.  The fused
// MGS steps are many_mgs_step_kernel + many_reduce_kernel on the columns still in the inner loop; the host reads the
// (inner + 3) x K coefficients of one H column per inner iteration in one copy, and the reorth pass runs masked to
// the columns whose test it meets.  The coefficients live in the hierarchy's gm_mgs scratch (gmres_mgs_scratch).
#pragma once

template <int K>
struct ManyGmres {
    amgb_hierarchy *h;
    ManyKrylov<K> M;
    long long n, npad;
    int mi;
    cudaStream_t s;

    ManyGmres(amgb_hierarchy *h_, int cyc, int mi_, bool dev)
        : h(h_), M(h_, cyc, dev), n(h_->levels[0].A.n_rows), npad(((h_->levels[0].A.n_rows + 2 + 31) / 32) * 32), mi(mi_),
          s(h_->stream) {}
    double *W(int j) const { return h->mgm_store + (size_t)j * npad * K; }
    double *Z(int j) const { return h->mgm_store + ((size_t)mi + 1 + j) * npad * K; }
    unsigned grid() const { return vec_grid(h->S, n); }
    double *slot(int i) const { return M.mw.norms2 + (size_t)i * K; }

    int to_level(const double *src, double *dst)      // original numbering -> level-0 numbering
    {
        if (h->order0 == nullptr) return copy(dst, src);
        many_pack_kernel<K><<<vec_grid(h->S, n * K), 256, 0, s>>>(src, K, K, h->order0, dst, n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    }
    int from_level(const double *src, double *dst)
    {
        if (h->pos0 == nullptr) return copy(dst, src);
        many_pack_kernel<K><<<vec_grid(h->S, n * K), 256, 0, s>>>(src, K, K, h->pos0, dst, n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    }
    int copy(double *dst, const double *src)          // copy_vec on the block
    {
        RET(M.copy(dst, src));
        h->launches++;
        return AMGB_OK;
    }
    // columns [c0, c0+w) of the caller's n x k block -> dst (original numbering, zero-padded); a host block is
    // staged through mw.io, a device block packed in place
    int load(const double *src, int32_t k, int c0, int w, double *dst)
    {
        const double *from = src + c0;
        long long ld = k;
        if (!M.dev) {
            const size_t wb = sizeof(double) * (size_t)w;
            CK(many_copy_2d(M.mw.io, wb, from, sizeof(double) * (size_t)k, wb, (size_t)n, cudaMemcpyHostToDevice, s));
            from = M.mw.io;
            ld = w;
        }
        many_pack_kernel<K><<<vec_grid(h->S, n * K), 256, 0, s>>>(from, ld, w, nullptr, dst, n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    }
    int store(const double *src, int32_t k, int c0, int w, double *dst)
    {
        many_unpack_kernel<K><<<vec_grid(h->S, n * w), 256, 0, s>>>(src, nullptr, M.dev ? dst + c0 : M.mw.io,
                                                                    M.dev ? k : w, 0, w, n);
        CK(cudaGetLastError());
        h->launches++;
        if (M.dev) return AMGB_OK;
        const size_t wb = sizeof(double) * (size_t)w;
        CK(many_copy_2d(dst + c0, sizeof(double) * (size_t)k, M.mw.io, wb, wb, (size_t)n, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return AMGB_OK;
    }
    int precond()                                      // V.x_home <- M V.b : one batched cycle from zero
    {
        return M.precond();
    }
    // z_q <- (I - 2 w_q w_q^T) z_q on the active columns, the inner products kept on the device (Gmres::reflect)
    int reflect(const double *w, double *z, unsigned active)
    {
        if (active == 0) return AMGB_OK;
        RET(M.dot(w, z, 2));
        many_axpy_ratio_kernel<K><<<grid(), 256, 0, s>>>(z, w, slot(2), slot(3), -2.0, active, n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    }
    // w_q = e_k1-shifted v_q + alpha_q e_k1, then w_q /= ||w_q|| on alpha.active (Gmres::make_w)
    int make_w(double *w, const double *v, long long k1, const ManyScalars &alpha)
    {
        if (alpha.active == 0) return AMGB_OK;
        many_hh_make_w_kernel<K><<<grid(), 256, 0, s>>>(w, v, k1, alpha, n);
        CK(cudaGetLastError());
        h->launches++;
        RET(M.dot(w, w, 0));
        RET(M.read(1));
        ManyScalars d = {};
        d.active = alpha.active;
        for (int q = 0; q < K; q++) d.v[q] = std::sqrt(M.got[(size_t)q]);
        many_div_kernel<K><<<grid(), 256, 0, s>>>(w, d, n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    }
};

// shape of the reflector store (doubles) for width K
static long long many_gmres_store_count(long long n, int mi, bool flex, int K)
{
    const long long npad = ((n + 2 + 31) / 32) * 32;
    return ((long long)mi + 1 + (flex ? mi : 0)) * npad * K;
}

// an allocation the device cannot satisfy -> AMGB_ENOTIMPL with the CUDA error cleared; other failures unchanged
static int many_gmres_oom(int rc)
{
    if (rc != AMGB_ECUDA) return rc;
    const cudaError_t e = cudaGetLastError();          // clears the allocation error
    if (e == cudaErrorMemoryAllocation || g_err.find(cudaGetErrorString(cudaErrorMemoryAllocation)) != std::string::npos)
        return fail(AMGB_ENOTIMPL, "solve_many gmres: the batched buffers do not fit in device memory");
    return rc;
}

// the level vectors and seven Krylov blocks of width K; a failed attempt frees what it allocated
template <int K>
static int many_gmres_prepare(amgb_hierarchy *h)
{
    ManyWidth &mw = h->many[many_index(K)];
    const bool had_lv = !mw.lv.empty();
    const size_t mark = h->allocs.size();
    const long long bytes = h->dev_bytes;
    const int rc = many_krylov_prepare<K>(h, 7);
    if (rc == AMGB_OK) return AMGB_OK;
    for (size_t i = mark; i < h->allocs.size(); i++) {
        void *p = h->allocs[i];
        cudaFree(p);
        if (mw.partials == p) mw.partials = nullptr;
        if (mw.io == p) mw.io = nullptr;
        if (mw.norms2 == p) { mw.norms2 = nullptr; mw.norms2_cap = 0; }
        for (double *&b : mw.kry)
            if (b == p) b = nullptr;
    }
    h->allocs.resize(mark);
    h->dev_bytes = bytes;
    if (!had_lv) mw.lv.clear();
    return many_gmres_oom(rc);
}

// a reflector store of at least `count` doubles (the previous one is freed first when it is too small)
static int many_gmres_store(amgb_hierarchy *h, long long count)
{
    if (h->mgm_count >= count) return AMGB_OK;
    if (h->mgm_store != nullptr) {
        CK(cudaStreamSynchronize(h->stream));          // nothing in flight may still use the store being replaced
        h->dfree(h->mgm_store);
        h->dev_bytes -= (long long)((sizeof(double) * (size_t)h->mgm_count + 255) & ~(size_t)255);
        h->mgm_count = 0;
    }
    RET(many_gmres_oom(h->dalloc(&h->mgm_store, count)));
    h->mgm_count = count;
    return AMGB_OK;
}

template <int K>
static int many_gmres_reserve(amgb_hierarchy *h, long long n, int mi, bool flex)
{
    RET(many_gmres_prepare<K>(h));
    return many_gmres_store(h, many_gmres_store_count(n, mi, flex, K));
}

static int many_gmres_reserve_width(amgb_hierarchy *h, int K, long long n, int mi, bool flex)
{
    switch (K) {
    case 2: return many_gmres_reserve<2>(h, n, mi, flex);
    case 4: return many_gmres_reserve<4>(h, n, mi, flex);
    default: return many_gmres_reserve<8>(h, n, mi, flex);
    }
}

// amgb_solve_gmres on columns [c0, c0+w) of the caller's n x k blocks
template <int K>
static int many_gmres_group(amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X, bool x0_zero,
                            bool dev, double tol, int mi, long long max_outer, bool flex, int32_t cycle, double *residuals,
                            int32_t max_residuals, int32_t *n_residuals, int32_t *info)
{
    ManyGmres<K> G(h, cycle, mi, dev);
    ManyKrylov<K> &M = G.M;
    ManyWidth &mw = M.mw;
    ManyLevel &V = M.V;
    const long long n = G.n;
    cudaStream_t s = h->stream;
    double *v = mw.kry[0], *xk = mw.kry[1], *bk = mw.kry[2], *upd = mw.kry[3];
    double *b_lvl = mw.kry[4], *lin = mw.kry[5], *lout = mw.kry[6];
    const double *mx = V.x_home;                       // the preconditioner's output
    const std::vector<double> ones((size_t)K, 1.0);
    CK(cudaMemcpyAsync(G.slot(3), ones.data(), sizeof(double) * K, cudaMemcpyHostToDevice, s));   // reflect's 1.0
    RET(G.load(B, k, c0, w, bk));
    if (x0_zero) RET(h->launch_count_fill(xk, n * K));
    else RET(G.load(X, k, c0, w, xk));
    RET(G.to_level(bk, b_lvl));

    // r = b - A x (then r = M r for the left-preconditioned method) -> the first reflectors' storage W(0)
    auto residual_to_w0 = [&]() -> int {
        RET(G.to_level(xk, lin));
        if (flex) {
            RET(many_spmv<K>(h, OP_RESID, M.A0, lin, b_lvl, lout));
            return G.from_level(lout, G.W(0));
        }
        RET(many_spmv<K>(h, OP_RESID, M.A0, lin, b_lvl, V.b));
        RET(G.precond());
        return G.from_level(mx, G.W(0));
    };
    std::vector<std::vector<double>> res((size_t)w);
    std::vector<double> normr((size_t)K, 0.0), scale((size_t)K, 1.0), bb((size_t)K, 0.0);
    RET(residual_to_w0());
    RET(M.dot(G.W(0), G.W(0), 0));
    RET(M.dot(bk, bk, 1));
    RET(M.read(2));
    unsigned need_scale = 0;
    for (int q = 0; q < w; q++) {
        normr[(size_t)q] = std::sqrt(M.got[(size_t)q]);
        res[(size_t)q].push_back(normr[(size_t)q]);                         // :165-167
        bb[(size_t)q] = M.got[(size_t)K + q];
        if (bb[(size_t)q] != 0.0) {                                          // :169-174 / _fgmres.py:171-174
            if (flex) scale[(size_t)q] = std::sqrt(bb[(size_t)q]);
            else need_scale |= 1u << q;
        }
    }
    if (need_scale != 0) {                                                   // ||M b||
        RET(G.copy(V.b, b_lvl));
        RET(G.precond());
        RET(G.from_level(mx, v));
        RET(M.dot(v, v, 0));
        RET(M.read(1));
        for (int q = 0; q < w; q++)
            if (need_scale & (1u << q)) scale[(size_t)q] = std::sqrt(M.got[(size_t)q]);
    }
    std::vector<int> status((size_t)w, -2), niter((size_t)w, 0);
    unsigned run = 0;                                                        // columns without a status
    for (int q = 0; q < w; q++) {
        if (normr[(size_t)q] < tol * scale[(size_t)q]) status[(size_t)q] = 0;   // :177-178
        else run |= 1u << q;
    }
    const int m2 = (int)std::min<long long>(n, (long long)mi + 1);           // leading rows of v the host needs
    std::vector<std::vector<double>> H((size_t)w), Q((size_t)w), g((size_t)w), y((size_t)w);
    std::vector<double> hv((size_t)m2);
    std::vector<int> last((size_t)w, mi - 1);                                // inner index each column ended at
    double *pin = nullptr;                                                   // m2 x K rows of v, then K norms
    CK(cudaHostAlloc((void **)&pin, sizeof(double) * ((size_t)m2 + 1) * K, cudaHostAllocDefault));
    struct PinGuard { double *p; ~PinGuard() { if (p) cudaFreeHost(p); } } pin_guard{pin};

    for (long long outer = 0; outer < max_outer && run != 0; outer++) {
        // first reflector from r: w = r; w[0] += sign(r[0]) ||r||; w /= ||w||          (:186-192)
        CK(cudaMemcpyAsync(pin, G.W(0), sizeof(double) * K, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        ManyScalars beta = {};
        beta.active = run;
        for (int q = 0; q < w; q++) {
            if (!(run & (1u << q))) continue;
            const double r0 = pin[q];
            beta.v[q] = (r0 == 0.0 ? 1.0 : r0 / std::fabs(r0)) * normr[(size_t)q];
        }
        RET(G.make_w(G.W(0), G.W(0), 0, beta));
        CK(cudaMemsetAsync(G.W(1), 0, sizeof(double) * (size_t)mi * (size_t)G.npad * K, s));   // W = zeros (:203)
        for (int q = 0; q < w; q++) {
            if (!(run & (1u << q))) continue;
            H[(size_t)q].assign((size_t)mi * mi, 0.0);
            Q[(size_t)q].assign((size_t)4 * mi, 0.0);
            g[(size_t)q].assign((size_t)mi + 1, 0.0);
            y[(size_t)q].assign((size_t)mi, 0.0);
            g[(size_t)q][0] = -beta.v[q];                                    // :208-209
            last[(size_t)q] = mi - 1;
        }
        unsigned in = run;                                                   // columns still in the inner loop
        for (int inner = 0; inner < mi && in != 0; inner++) {
            many_hh_unit_reflect_kernel<K><<<G.grid(), 256, 0, s>>>(v, G.W(inner), inner, in, n);   // :214-215
            CK(cudaGetLastError());
            h->launches++;
            for (int j = inner - 1; j >= 0; j--) RET(G.reflect(G.W(j), v, in));                     // :219
            if (flex) {                                                      // _fgmres.py:221-230
                RET(G.to_level(v, V.b));
                RET(G.precond());
                RET(G.from_level(mx, G.Z(inner)));
                RET(many_spmv<K>(h, OP_SPMV, M.A0, mx, nullptr, lout));
                RET(G.from_level(lout, v));
            } else {                                                         // :222-225
                RET(G.to_level(v, lin));
                RET(many_spmv<K>(h, OP_SPMV, M.A0, lin, nullptr, V.b));
                RET(G.precond());
                RET(G.from_level(mx, v));
            }
            for (int j = 0; j <= inner; j++) RET(G.reflect(G.W(j), v, in));                         // :235
            const bool tail = inner != n - 1;
            if (tail) {                                                      // ||v[inner+1:]||^2 (:239-240)
                many_sumsq_from_kernel<K><<<sumsq_blocks(h->S), 256, 0, s>>>(v, inner + 1, n, mw.partials);
                CK(cudaGetLastError());
                many_reduce_kernel<K><<<1, 1024, 0, s>>>(mw.partials, sumsq_blocks(h->S), G.slot(0));
                CK(cudaGetLastError());
                h->launches += 2;
                CK(cudaMemcpyAsync(pin + (size_t)m2 * K, G.slot(0), sizeof(double) * K, cudaMemcpyDeviceToHost, s));
            }
            CK(cudaMemcpyAsync(pin, v, sizeof(double) * (size_t)m2 * K, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            ManyScalars alpha_w = {};                                        // columns that get a next reflector
            std::vector<std::vector<double>> hvs((size_t)w);
            for (int q = 0; q < w; q++) {
                if (!(in & (1u << q))) continue;
                std::vector<double> &hq = hvs[(size_t)q];
                hq.resize((size_t)m2);
                for (int r = 0; r < m2; r++) hq[(size_t)r] = pin[(size_t)r * K + q];
                if (tail) {                                                  // :244-263
                    double alpha = std::sqrt(pin[(size_t)m2 * K + q]);
                    if (alpha != 0.0) {
                        const double v0 = hq[(size_t)inner + 1];
                        alpha = (v0 == 0.0 ? 1.0 : v0 / std::fabs(v0)) * alpha;
                        if (inner < mi - 1) { alpha_w.v[q] = alpha; alpha_w.active |= 1u << q; }
                        hq[(size_t)inner + 1] = -alpha;
                        for (int r = inner + 2; r < m2; r++) hq[(size_t)r] = 0.0;
                    }
                }
            }
            RET(G.make_w(G.W(inner + 1), v, inner + 1, alpha_w));
            for (int q = 0; q < w; q++) {
                if (!(in & (1u << q))) continue;
                std::vector<double> &hq = hvs[(size_t)q], &Qq = Q[(size_t)q], &gq = g[(size_t)q];
                for (int rot = 0; rot < inner; rot++) {                      // apply_givens (krylov.h:171-186)
                    const double xt = hq[(size_t)rot];
                    hq[(size_t)rot] = Qq[(size_t)4 * rot] * xt + Qq[(size_t)4 * rot + 1] * hq[(size_t)rot + 1];
                    hq[(size_t)rot + 1] = Qq[(size_t)4 * rot + 2] * xt + Qq[(size_t)4 * rot + 3] * hq[(size_t)rot + 1];
                }
                if (tail && hq[(size_t)inner + 1] != 0.0) {                  // :276-291
                    double c, sn, rr;
                    lartg(hq[(size_t)inner], hq[(size_t)inner + 1], &c, &sn, &rr);
                    double *qr = &Qq[(size_t)4 * inner];
                    qr[0] = c; qr[1] = sn; qr[2] = -sn; qr[3] = c;
                    const double g0 = gq[(size_t)inner], g1 = gq[(size_t)inner + 1];
                    gq[(size_t)inner] = c * g0 + sn * g1;
                    gq[(size_t)inner + 1] = -sn * g0 + c * g1;
                    hq[(size_t)inner] = c * hq[(size_t)inner] + sn * hq[(size_t)inner + 1];
                    hq[(size_t)inner + 1] = 0.0;
                }
                for (int r = 0; r < mi; r++) H[(size_t)q][(size_t)r * mi + inner] = hq[(size_t)r];   // H[:, inner] (:295)
                if (!flex) niter[(size_t)q]++;                               // :297
                if (inner < mi - 1) {                                        // :301-305
                    normr[(size_t)q] = std::fabs(gq[(size_t)inner + 1]);
                    if (normr[(size_t)q] < tol * scale[(size_t)q]) {         // (fgmres: before niter += 1)
                        last[(size_t)q] = inner;
                        in &= ~(1u << q);
                        continue;
                    }
                    res[(size_t)q].push_back(normr[(size_t)q]);
                }
                if (flex) niter[(size_t)q]++;                                // _fgmres.py:306
            }
        }
        // per column: solve H[0:k,0:k] y = g[0:k] (upper triangular), k = inner + 1
        int kmax = 0;
        for (int q = 0; q < w; q++) {
            if (!(run & (1u << q))) continue;
            const int kq = last[(size_t)q] + 1;
            const std::vector<double> &Hq = H[(size_t)q], &gq = g[(size_t)q];
            std::vector<double> &yq = y[(size_t)q];
            for (int i = kq - 1; i >= 0; i--) {
                double acc = gq[(size_t)i];
                for (int j = i + 1; j < kq; j++) acc -= Hq[(size_t)i * mi + j] * yq[(size_t)j];
                yq[(size_t)i] = acc / Hq[(size_t)i * mi + i];
            }
            kmax = std::max(kmax, kq);
        }
        auto coef = [&](int j) {                                             // y_j of the columns with k > j
            ManyScalars c = {};
            for (int q = 0; q < w; q++)
                if ((run & (1u << q)) && last[(size_t)q] + 1 > j) { c.v[q] = y[(size_t)q][(size_t)j]; c.active |= 1u << q; }
            return c;
        };
        if (flex) {                                                          // update = Z[:, 0:k] y (_fgmres.py:321)
            many_scale_kernel<K><<<G.grid(), 256, 0, s>>>(upd, coef(0), G.Z(0), n);
            CK(cudaGetLastError());
            h->launches++;
            for (int j = 1; j < kmax; j++) {
                const ManyScalars c = coef(j);
                ManyAxpby a = {};
                for (int q = 0; q < K; q++) { a.a[q] = c.v[q]; a.b[q] = 1.0; }
                a.active = c.active;
                many_axpby_kernel<K><<<vec_grid(h->S, n), 256, 0, s>>>(a, G.Z(j), upd, n);
                CK(cudaGetLastError());
                h->launches++;
            }
        } else {                                                             // householder_hornerscheme (:321-322)
            RET(h->launch_count_fill(upd, n * K));
            for (int j = kmax - 1; j >= 0; j--) {
                const ManyScalars c = coef(j);
                many_add_at_kernel<K><<<1, 1, 0, s>>>(upd, j, c);
                CK(cudaGetLastError());
                h->launches++;
                RET(G.reflect(G.W(j), upd, c.active));
            }
        }
        const std::vector<double> one((size_t)K, 1.0);
        RET(M.axpby(one.data(), upd, one.data(), xk, run));                 // x = x + update (:324)
        RET(residual_to_w0());                                               // :325-328
        RET(M.dot(G.W(0), G.W(0), 0));
        many_maxratio_kernel<K><<<sumsq_blocks(h->S), 256, 0, s>>>(upd, xk, n, mw.partials);   // :339-346
        CK(cudaGetLastError());
        many_reduce_max_kernel<K><<<1, 1024, 0, s>>>(mw.partials, sumsq_blocks(h->S), G.slot(1));
        CK(cudaGetLastError());
        h->launches += 2;
        RET(M.read(2));
        for (int q = 0; q < w; q++) {
            if (!(run & (1u << q))) continue;
            normr[(size_t)q] = std::sqrt(M.got[(size_t)q]);
            res[(size_t)q].push_back(normr[(size_t)q]);                      // :335-336
            const double change = M.got[(size_t)K + q];
            if (change >= 0.0 && change < 1e-12) { status[(size_t)q] = -1; run &= ~(1u << q); continue; }
            if (normr[(size_t)q] < tol * scale[(size_t)q]) { status[(size_t)q] = 0; run &= ~(1u << q); }   // :349-350
        }
    }
    for (int q = 0; q < w; q++)
        if (status[(size_t)q] == -2) status[(size_t)q] = niter[(size_t)q];  // :354
    RET(G.store(xk, k, c0, w, X));
    for (int q = 0; q < w; q++) {
        const std::vector<double> &rq = res[(size_t)q];
        const size_t nres = std::min<size_t>(rq.size(), (size_t)std::max(max_residuals, 0));
        if (residuals != nullptr)
            for (size_t t = 0; t < nres; t++) residuals[t * (size_t)k + c0 + q] = rq[t];
        if (n_residuals != nullptr) n_residuals[c0 + q] = (int32_t)rq.size();
        if (info != nullptr) info[c0 + q] = status[(size_t)q];
    }
    return AMGB_OK;
}

// amgb_solve_gmres(..., AMGB_FLAG_MGS) on columns [c0, c0+w) of the caller's n x k blocks: gmres_mgs of
// abi_krylov.cuh restated on n x K blocks in the level-0 numbering, the basis in the store's W slots
template <int K>
static int many_gmres_mgs_group(amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X, bool x0_zero,
                                bool dev, double tol, int mi, long long max_outer, bool reorth, int32_t cycle,
                                double *residuals, int32_t max_residuals, int32_t *n_residuals, int32_t *info)
{
    ManyGmres<K> G(h, cycle, mi, dev);
    ManyKrylov<K> &M = G.M;
    ManyWidth &mw = M.mw;
    ManyLevel &V = M.V;
    const long long n = G.n;
    cudaStream_t s = h->stream;
    const int nb = sumsq_blocks(h->S);
    double *xk = mw.kry[1], *bk = mw.kry[2], *upd = mw.kry[3];
    double *mv = V.x_home;                             // the preconditioner's output, MGS's work vector v
    double *coef = h->gm_mgs, *coef2 = h->gm_mgs + (size_t)(mi + 3) * K, *sq_parts = h->gm_mgs + (size_t)2 * (mi + 3) * K;
    RET(M.load(B, k, c0, w, bk));
    if (x0_zero) RET(h->launch_count_fill(xk, n * K));
    else RET(M.load(X, k, c0, w, xk));

    std::vector<double> normMb((size_t)K, 1.0), normr((size_t)K, 0.0);      // :204-207, ||M b|| before r
    RET(M.dot(bk, bk, 0));
    RET(M.read(1));
    unsigned need = 0;
    for (int q = 0; q < w; q++)
        if (M.got[(size_t)q] != 0.0) need |= 1u << q;
    if (need != 0) {
        RET(G.copy(V.b, bk));
        RET(M.precond());
        RET(M.dot(mv, mv, 0));
        RET(M.read(1));
        for (int q = 0; q < w; q++)
            if (need & (1u << q)) normMb[(size_t)q] = std::sqrt(M.got[(size_t)q]);
    }
    auto residual = [&]() -> int {                                           // mv = M (b - A x)   (:192-195)
        RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, V.b));
        return M.precond();
    };
    RET(residual());
    RET(M.dot(mv, mv, 0));
    RET(M.read(1));
    std::vector<std::vector<double>> res((size_t)w);
    std::vector<int> status((size_t)w, -2), niter((size_t)w, 0);
    unsigned run = 0;                                                        // columns without a status
    for (int q = 0; q < w; q++) {
        normr[(size_t)q] = std::sqrt(M.got[(size_t)q]);
        res[(size_t)q].push_back(normr[(size_t)q]);                          // :197-198
        if (normr[(size_t)q] < tol * normMb[(size_t)q]) status[(size_t)q] = 0;   // :209-210
        else run |= 1u << q;
    }

    // gmres_mgs's mgs_pass on the columns in `active`: slot j of c holds the K coefficients of V_j
    auto mgs_pass = [&](int inner, double *c, bool norms, unsigned active) -> int {
        for (int j = 0; j <= inner + 1; j++) {
            const bool last = j == inner + 1, sq = norms && (j == 0 || last);
            many_mgs_step_kernel<K><<<nb, 256, 0, s>>>(mv, j > 0 ? G.W(j - 1) : nullptr, c + (size_t)(j > 0 ? j - 1 : 0) * K,
                                                       last ? nullptr : G.W(j), active, n, last ? nullptr : mw.partials,
                                                       sq ? sq_parts : nullptr);
            CK(cudaGetLastError());
            h->launches++;
            if (!last) {
                many_reduce_kernel<K><<<1, 1024, 0, s>>>(mw.partials, nb, c + (size_t)j * K);
                CK(cudaGetLastError());
                h->launches++;
            }
            if (sq) {
                many_reduce_kernel<K><<<1, 1024, 0, s>>>(sq_parts, nb, c + (size_t)(inner + (last ? 2 : 1)) * K);
                CK(cudaGetLastError());
                h->launches++;
            }
        }
        return AMGB_OK;
    };
    auto scale_next = [&](int inner, unsigned active) -> int {               // V[inner+1] = v / normv (:268-269)
        many_mgs_scale_kernel<K><<<G.grid(), 256, 0, s>>>(G.W(inner + 1), mv, coef + (size_t)(inner + 2) * K, active, n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    };
    std::vector<std::vector<double>> H((size_t)w), Q((size_t)w), g((size_t)w), y((size_t)w), hvs((size_t)w);
    std::vector<int> last((size_t)w, mi - 1);                                // inner index each column ended at
    double *col = nullptr;                                                   // (inner + 3) x K coefficients
    CK(cudaHostAlloc((void **)&col, sizeof(double) * ((size_t)mi + 3) * K, cudaHostAllocDefault));
    struct PinGuard { double *p; ~PinGuard() { if (p) cudaFreeHost(p); } } pin_guard{col};

    for (long long outer = 0; outer < max_outer && run != 0; outer++) {
        ManyScalars inv = {};                                                // V[0] = r * (1 / normr) (:225-226)
        inv.active = run;
        for (int q = 0; q < w; q++)
            if (run & (1u << q)) inv.v[q] = 1.0 / normr[(size_t)q];
        many_scale_kernel<K><<<G.grid(), 256, 0, s>>>(G.W(0), inv, mv, n);
        CK(cudaGetLastError());
        h->launches++;
        for (int q = 0; q < w; q++) {
            if (!(run & (1u << q))) continue;
            H[(size_t)q].assign((size_t)mi * mi, 0.0);
            Q[(size_t)q].assign((size_t)4 * mi, 0.0);
            g[(size_t)q].assign((size_t)mi + 1, 0.0);
            y[(size_t)q].assign((size_t)mi, 0.0);
            hvs[(size_t)q].assign((size_t)mi + 2, 0.0);
            g[(size_t)q][0] = normr[(size_t)q];                              // :230-231
            last[(size_t)q] = mi - 1;
        }
        unsigned in = run;                                                   // columns still in the inner loop
        for (int inner = 0; inner < mi && in != 0; inner++) {
            RET(many_spmv<K>(h, OP_SPMV, M.A0, G.W(inner), nullptr, V.b));  // v = M (A V[inner])  (:237)
            RET(M.precond());
            RET(mgs_pass(inner, coef, true, in));                            // :238-258
            if (!reorth) RET(scale_next(inner, in));
            CK(cudaMemcpyAsync(col, coef, sizeof(double) * ((size_t)inner + 3) * K, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            unsigned ro = 0;                                                 // columns that take the reorth pass
            for (int q = 0; q < w; q++) {
                if (!(in & (1u << q))) continue;
                std::vector<double> &hq = hvs[(size_t)q];
                for (int r = 0; r <= inner; r++) hq[(size_t)r] = col[(size_t)r * K + q];
                const double normv_old = std::sqrt(col[(size_t)(inner + 1) * K + q]);
                const double normv = std::sqrt(col[(size_t)(inner + 2) * K + q]);
                hq[(size_t)inner + 1] = normv;                               // H[inner, inner+1] (:257)
                if (reorth && normv_old == normv_old + 0.001 * normv) ro |= 1u << q;   // :260
            }
            if (ro != 0) {                                                   // :261-266
                RET(mgs_pass(inner, coef2, false, ro));
                CK(cudaMemcpyAsync(col, coef2, sizeof(double) * ((size_t)inner + 1) * K, cudaMemcpyDeviceToHost, s));
                CK(cudaStreamSynchronize(s));
                for (int q = 0; q < w; q++)
                    if (ro & (1u << q))
                        for (int r = 0; r <= inner; r++) hvs[(size_t)q][(size_t)r] = hvs[(size_t)q][(size_t)r] + col[(size_t)r * K + q];
            }
            if (reorth) RET(scale_next(inner, in));
            for (int q = 0; q < w; q++) {
                if (!(in & (1u << q))) continue;
                std::vector<double> &hq = hvs[(size_t)q], &Qq = Q[(size_t)q], &gq = g[(size_t)q];
                for (int rot = 0; rot < inner; rot++) {                      // apply_givens (:13-39, :272-273)
                    const double xt = hq[(size_t)rot];
                    hq[(size_t)rot] = Qq[(size_t)4 * rot] * xt + Qq[(size_t)4 * rot + 1] * hq[(size_t)rot + 1];
                    hq[(size_t)rot + 1] = Qq[(size_t)4 * rot + 2] * xt + Qq[(size_t)4 * rot + 3] * hq[(size_t)rot + 1];
                }
                if (inner != n - 1 && hq[(size_t)inner + 1] != 0.0) {        // :278-290
                    double c, sn, rr;
                    lartg(hq[(size_t)inner], hq[(size_t)inner + 1], &c, &sn, &rr);
                    double *qr = &Qq[(size_t)4 * inner];
                    qr[0] = c; qr[1] = sn; qr[2] = -sn; qr[3] = c;
                    const double g0 = gq[(size_t)inner], g1 = gq[(size_t)inner + 1];
                    gq[(size_t)inner] = c * g0 + sn * g1;
                    gq[(size_t)inner + 1] = -sn * g0 + c * g1;
                    hq[(size_t)inner] = c * hq[(size_t)inner] + sn * hq[(size_t)inner + 1];
                    hq[(size_t)inner + 1] = 0.0;
                }
                for (int r = 0; r < mi; r++) H[(size_t)q][(size_t)r * mi + inner] = hq[(size_t)r];
                niter[(size_t)q]++;                                          // :292
                if (inner < mi - 1) {                                        // :296-302
                    normr[(size_t)q] = std::fabs(gq[(size_t)inner + 1]);
                    if (normr[(size_t)q] < tol * normMb[(size_t)q]) {
                        last[(size_t)q] = inner;
                        in &= ~(1u << q);
                        continue;
                    }
                    res[(size_t)q].push_back(normr[(size_t)q]);
                }
            }
        }
        // per column: solve H[0:k,0:k].T y = g[0:k] (upper triangular as stored), k = inner + 1 (:312)
        int kmax = 0;
        for (int q = 0; q < w; q++) {
            if (!(run & (1u << q))) continue;
            const int kq = last[(size_t)q] + 1;
            const std::vector<double> &Hq = H[(size_t)q], &gq = g[(size_t)q];
            std::vector<double> &yq = y[(size_t)q];
            for (int i = kq - 1; i >= 0; i--) {
                double acc = gq[(size_t)i];
                for (int j = i + 1; j < kq; j++) acc -= Hq[(size_t)i * mi + j] * yq[(size_t)j];
                yq[(size_t)i] = acc / Hq[(size_t)i * mi + i];
            }
            kmax = std::max(kmax, kq);
        }
        auto coef_y = [&](int j) {                                           // y_j of the columns with k > j
            ManyScalars c = {};
            for (int q = 0; q < w; q++)
                if ((run & (1u << q)) && last[(size_t)q] + 1 > j) { c.v[q] = y[(size_t)q][(size_t)j]; c.active |= 1u << q; }
            return c;
        };
        many_scale_kernel<K><<<G.grid(), 256, 0, s>>>(upd, coef_y(0), G.W(0), n);   // update = V[:k].T y (:313)
        CK(cudaGetLastError());
        h->launches++;
        for (int j = 1; j < kmax; j++) {
            const ManyScalars c = coef_y(j);
            ManyAxpby a = {};
            for (int q = 0; q < K; q++) { a.a[q] = c.v[q]; a.b[q] = 1.0; }
            a.active = c.active;
            many_axpby_kernel<K><<<vec_grid(h->S, n), 256, 0, s>>>(a, G.W(j), upd, n);
            CK(cudaGetLastError());
            h->launches++;
        }
        const std::vector<double> one((size_t)K, 1.0);
        RET(M.axpby(one.data(), upd, one.data(), xk, run));                 // x = x + update (:314)
        RET(residual());                                                     // :315-319
        RET(M.dot(mv, mv, 0));
        many_maxratio_kernel<K><<<nb, 256, 0, s>>>(upd, xk, n, mw.partials); // :328-334
        CK(cudaGetLastError());
        many_reduce_max_kernel<K><<<1, 1024, 0, s>>>(mw.partials, nb, G.slot(1));
        CK(cudaGetLastError());
        h->launches += 2;
        RET(M.read(2));
        for (int q = 0; q < w; q++) {
            if (!(run & (1u << q))) continue;
            normr[(size_t)q] = std::sqrt(M.got[(size_t)q]);
            res[(size_t)q].push_back(normr[(size_t)q]);                      // :324-325
            const double change = M.got[(size_t)K + q];
            if (change >= 0.0 && change < 1e-12) { status[(size_t)q] = -1; run &= ~(1u << q); continue; }
            if (normr[(size_t)q] < tol * normMb[(size_t)q]) { status[(size_t)q] = 0; run &= ~(1u << q); }   // :337-338
        }
    }
    for (int q = 0; q < w; q++)
        if (status[(size_t)q] == -2) status[(size_t)q] = niter[(size_t)q];  // :342
    RET(M.store(xk, k, c0, w, X));
    for (int q = 0; q < w; q++) {
        const std::vector<double> &rq = res[(size_t)q];
        const size_t nres = std::min<size_t>(rq.size(), (size_t)std::max(max_residuals, 0));
        if (residuals != nullptr)
            for (size_t t = 0; t < nres; t++) residuals[t * (size_t)k + c0 + q] = rq[t];
        if (n_residuals != nullptr) n_residuals[c0 + q] = (int32_t)rq.size();
        if (info != nullptr) info[c0 + q] = status[(size_t)q];
    }
    return AMGB_OK;
}

// one group of amgb_solve_many_gmres at width K
template <int K>
static int many_gmres_run(amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X, int32_t flags,
                          bool dev, double tol, int mi, long long max_outer, int32_t cycle, double *residuals,
                          int32_t max_residuals, int32_t *n_residuals, int32_t *info)
{
    const bool x0_zero = (flags & AMGB_FLAG_X0_ZERO) != 0;
    if (flags & AMGB_FLAG_MGS)
        return many_gmres_mgs_group<K>(h, k, c0, w, B, X, x0_zero, dev, tol, mi, max_outer, (flags & AMGB_FLAG_REORTH) != 0,
                                       cycle, residuals, max_residuals, n_residuals, info);
    return many_gmres_group<K>(h, k, c0, w, B, X, x0_zero, dev, tol, mi, max_outer, (flags & AMGB_FLAG_FLEXIBLE) != 0,
                               cycle, residuals, max_residuals, n_residuals, info);
}

extern "C" int amgb_solve_many_gmres(amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host, double tol,
                                     int32_t restart, int32_t maxiter, int32_t cycle, int32_t flags, double *residuals,
                                     int32_t max_residuals, int32_t *n_residuals, int32_t *info)
{
    RET(check_many_args(h, k, cycle, 1, B_host, X_host));
    if (restart < 0) return fail(AMGB_EINVAL, "restart < 0");
    RET(check_gmres_flags(flags));
    const long long n = h->levels[0].A.n_rows;
    if (n < 2) return fail(AMGB_EINVAL, "gmres: n < 2 is the caller's closed form (b / A[0,0])");
    const bool flex = (flags & AMGB_FLAG_FLEXIBLE) != 0;
    CallerIo io(h, flags);
    RET(io.begin(B_host, X_host));
    // _gmres_householder.py:129-149, as amgb_solve_gmres
    long long max_outer, max_inner;
    if (restart > 0) {
        max_outer = maxiter > 0 ? maxiter : 1;
        max_inner = std::min<long long>(restart, n);
    } else {
        max_outer = 1;
        max_inner = maxiter > 0 ? std::min<long long>(maxiter, n) : std::min<long long>(n, 40);
    }
    const int mi = (int)max_inner;
    h->launches = 0;
    // the widest width the columns need whose buffers fit; the last group of a call may be narrower
    int Kw = 0;
    for (int K = many_width(std::min(k, 8)); K >= 2 && Kw == 0; K /= 2) {
        int rc = many_gmres_reserve_width(h, K, n, mi, flex);
        const int rem = k % K;
        if (rc == AMGB_OK && rem != 0 && many_width(rem) < K) rc = many_gmres_reserve_width(h, many_width(rem), n, mi, flex);
        if (rc == AMGB_OK) Kw = K;
        else if (rc != AMGB_ENOTIMPL) return rc;
    }
    if (Kw == 0) return fail(AMGB_ENOTIMPL, "solve_many gmres: no batched width fits in device memory");
    if (flags & AMGB_FLAG_MGS) RET(many_gmres_oom(gmres_mgs_scratch(h, mi, Kw)));
    for (int c0 = 0; c0 < k; c0 += Kw) {
        const int w = std::min(Kw, k - c0);
        switch (many_width(w)) {
        case 2: RET(many_gmres_run<2>(h, k, c0, w, B_host, X_host, flags, io.dev, tol, mi, max_outer, cycle, residuals,
                                       max_residuals, n_residuals, info)); break;
        case 4: RET(many_gmres_run<4>(h, k, c0, w, B_host, X_host, flags, io.dev, tol, mi, max_outer, cycle, residuals,
                                       max_residuals, n_residuals, info)); break;
        default: RET(many_gmres_run<8>(h, k, c0, w, B_host, X_host, flags, io.dev, tol, mi, max_outer, cycle, residuals,
                                        max_residuals, n_residuals, info)); break;
        }
    }
    h->last_launches = h->launches;
    return io.end();
}
