// abi_krylov.cuh -- part of engine.cu's translation unit (included there): the GPU-resident Krylov accelerators
// amgb_solve_cg and amgb_solve_gmres (SURVEY.md 8(f)-1; Householder, flexible and modified Gram-Schmidt GMRES).  Uses the helpers and the amgb_hierarchy type defined above its
// include point; not a stand-alone header.
#pragma once

// ------------------------------------------------------------------------------------------
// GPU-resident preconditioned CG (SURVEY.md 8(f)-1): ml.solve(accel='cg') with every vector in HBM.
// Restates pyamg/krylov/_cg.py:97-196 (criteria 'rr': stop when ||r|| < tol ||b||; r recomputed from
// b - A x every 8th step, updated by r -= alpha A p otherwise; aborts on p'Ap < 0 or r'z < 0) with
// M = one multigrid cycle from x0 = 0 (MultilevelSolver.aspreconditioner, multilevel.py:355-396).
// r lives in the level-0 rhs buffer (the cycle never writes it), z is the cycle's level-0 iterate.
// Dot products are two-stage with a fixed grid (bit-reproducible); their values are read on the host
// once per iteration -- two tiny synchronisations against a whole cycle.
// ------------------------------------------------------------------------------------------
static int dev_dot(amgb_hierarchy *h, const double *x, const double *y, long long n, double *out_host)
{
    dot_partials_kernel<<<sumsq_blocks(h->S), 256, 0, h->stream>>>(x, y, n, h->sumsq_parts);
    CK(cudaGetLastError());
    reduce_partials_kernel<<<1, 1024, 0, h->stream>>>(h->sumsq_parts, sumsq_blocks(h->S), h->norms2);
    CK(cudaGetLastError());
    h->launches += 2;
    CK(cudaMemcpyAsync(h->norm_host, h->norms2, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *out_host = h->norm_host[0];
    return AMGB_OK;
}

static int dev_axpby(amgb_hierarchy *h, double a, const double *x, double b, double *y, long long n)
{
    if (n <= 0) return AMGB_OK;
    axpby_kernel<<<vec_grid(h->S, n), 256, 0, h->stream>>>(a, x, b, y, n);
    CK(cudaGetLastError());
    h->launches++;
    return AMGB_OK;
}

extern "C" int amgb_solve_cg(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t maxiter,
                             int32_t cycle, int32_t flags, double *residuals, int32_t *n_residuals, int32_t *info)
{
    RET(check_cycle_args(h, cycle, 1));
    if (b_host == nullptr || x_host == nullptr) return fail(AMGB_EINVAL, "null host vector");
    if (maxiter < 1) return fail(AMGB_EINVAL, "Number of iterations must be positive");    // _cg.py:95-96
    CK(cudaSetDevice(h->device));
    CallerIo io(h, flags);
    RET(io.begin(b_host, x_host));
    Level &L0 = h->levels[0];
    const long long n = L0.A.n_rows;
    cudaStream_t s = h->stream;
    h->launches = 0;
    if (h->kry[0] == nullptr)
        for (int k = 0; k < 4; k++) RET(h->dalloc(&h->kry[k], n + 2));
    double *xk = h->kry[0], *p = h->kry[1], *Ap = h->kry[2], *bk = h->kry[3];
    double *r = L0.b;                                     // CG residual = rhs of the preconditioner
    // b -> bk, x0 -> xk (level-0 numbering)
    RET(load_level0(h, b_host, (flags & AMGB_FLAG_X0_ZERO) ? nullptr : x_host, io.in_kind()));
    CK(cudaMemcpyAsync(bk, L0.b, sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(xk, L0.x, sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, s));
    auto precond = [&]() -> int {                         // z = M r: one cycle from zero on (L0.x, L0.b = r)
        L0.x = L0.x_home;
        RET(h->launch_count_fill(L0.x, n));
        return h->one_iteration(cycle, 1);
    };
    double normb2 = 0, rz = 0, rr = 0, pAp = 0;
    RET(dev_dot(h, bk, bk, n, &normb2));
    double normb = std::sqrt(normb2);
    if (normb == 0.0) normb = 1.0;
    RET(h->spmv(OP_RESID, L0.A, xk, bk, r));              // r = b - A x        (:99)
    RET(precond());                                       // z = M r            (:100)
    CK(cudaMemcpyAsync(p, L0.x, sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, s));   // p = z (:101)
    RET(dev_dot(h, r, L0.x, n, &rz));                     // rz = <r, z>        (:102)
    RET(dev_dot(h, r, r, n, &rr));
    std::vector<double> res;
    res.push_back(std::sqrt(rr));                         // residuals[:] = [normr] (:104-106)
    const double rtol = tol * normb;                      // criteria 'rr'      (:114-115)
    int it = 0, status = -2;
    if (res.back() < rtol) status = 0;                    // :133-134
    while (status == -2) {
        RET(h->spmv(OP_SPMV, L0.A, p, nullptr, Ap));      // Ap = A p           (:142)
        const double rz_old = rz;
        RET(dev_dot(h, Ap, p, n, &pAp));                  // curvature of A     (:145-148)
        if (pAp < 0.0) { status = -1; break; }
        const double alpha = rz / pAp;                    // :150
        RET(dev_axpby(h, alpha, p, 1.0, xk, n));          // x += alpha p       (:151)
        if ((it % 8) != 0 && it > 0) {
            RET(dev_axpby(h, -alpha, Ap, 1.0, r, n));     // r -= alpha Ap      (:153-154)
        } else {
            RET(h->spmv(OP_RESID, L0.A, xk, bk, r));      // r = b - A x        (:155-156)
        }
        RET(precond());                                   // z = M r            (:158)
        RET(dev_dot(h, r, L0.x, n, &rz));                 // :159
        if (rz < 0.0) { status = -1; break; }             // curvature of M     (:161-163)
        const double beta = rz / rz_old;                  // :165
        RET(dev_axpby(h, 1.0, L0.x, beta, p, n));         // p = beta p + z     (:166-167)
        it++;
        RET(dev_dot(h, r, r, n, &rr));
        res.push_back(std::sqrt(rr));                     // :171-174
        if (res.back() < rtol) { status = 0; break; }     // :190-191
        if (it == maxiter) { status = it; break; }        // :193-194
    }
    // x out (original numbering)
    CK(cudaMemcpyAsync(L0.x_home, xk, sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, s));
    L0.x = L0.x_home;
    RET(store_level0(h, x_host, io.out_kind()));
    RET(io.end());
    if (!io.dev) CK(cudaStreamSynchronize(s));
    if (residuals != nullptr)
        for (size_t k = 0; k < res.size() && k < (size_t)maxiter + 1; k++) residuals[k] = res[k];
    if (n_residuals != nullptr) *n_residuals = (int32_t)res.size();
    if (info != nullptr) *info = status;
    h->last_launches = h->launches;
    return AMGB_OK;
}

// ------------------------------------------------------------------------------------------
// GPU-resident Householder GMRES and flexible GMRES (SURVEY.md 8(f)-1): ml.solve(accel='gmres' | 'fgmres') with
// every long vector in HBM.  Restates pyamg/krylov/_gmres_householder.py:21-360 (what pyamg.krylov.gmres resolves
// to, LEFT preconditioning, stop on the preconditioned residual vs ||M b||) and pyamg/krylov/_fgmres.py:17-345
// (RIGHT preconditioning, the preconditioned directions are stored) with the native helpers of
// pyamg/amg_core/krylov.h (apply_householders :37-62, householder_hornerscheme :106-135, apply_givens :158-187);
// M = one multigrid cycle from a zero guess (aspreconditioner, multilevel.py:355-396).
// The reflectors single out the LEADING entries of the vectors, so the Krylov vectors live in the ORIGINAL
// numbering; they are gathered into the level-0 (wave-major) numbering around the SpMV + cycle.  The small
// Hessenberg / Givens / back-substitution work stays on the host (<= 41 x 41); per inner iteration the host reads
// max_inner + 1 leading entries of v and two scalars.
// ------------------------------------------------------------------------------------------
namespace {
struct Gmres {
    amgb_hierarchy *h;
    long long n, npad;
    int cycle;
    cudaStream_t s;
    Level &L0;
    Gmres(amgb_hierarchy *h_, int cyc) : h(h_), n(h_->levels[0].A.n_rows), npad(((h_->levels[0].A.n_rows + 2 + 31) / 32) * 32),
                                         cycle(cyc), s(h_->stream), L0(h_->levels[0]) {}
    double *W(int j) const { return h->gm_W + (size_t)j * npad; }
    double *Z(int j) const { return h->gm_Z + (size_t)j * npad; }
    unsigned grid() const { return vec_grid(h->S, n); }

    int to_level(const double *src, double *dst)      // original numbering -> level-0 numbering
    {
        if (h->order0 == nullptr) return h->copy_vec(dst, src, n);
        return h->gather(src, h->order0, dst, n);
    }
    int from_level(const double *src, double *dst)
    {
        if (h->pos0 == nullptr) return h->copy_vec(dst, src, n);
        return h->gather(src, h->pos0, dst, n);
    }
    int precond()                                      // L0.x <- M L0.b : one cycle from zero
    {
        L0.x = L0.x_home;
        RET(h->launch_count_fill(L0.x, n));
        return h->one_iteration(cycle, 1);
    }
    int read(const double *dev, double *host, int count)
    {
        CK(cudaMemcpyAsync(h->norm_host, dev, sizeof(double) * (size_t)std::min(count, 2), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        for (int k = 0; k < std::min(count, 2); k++) host[k] = h->norm_host[k];
        return AMGB_OK;
    }
    int dot(const double *x, const double *y, double *out)
    {
        RET(h->dot_to(x, y, n, h->gm_s));
        return read(h->gm_s, out, 1);
    }
    int sumsq_from(const double *x, long long start, double *out)
    {
        sumsq_from_partials_kernel<<<sumsq_blocks(h->S), 256, 0, s>>>(x, start, n, h->sumsq_parts);
        CK(cudaGetLastError());
        reduce_partials_kernel<<<1, 1024, 0, s>>>(h->sumsq_parts, sumsq_blocks(h->S), h->gm_s);
        CK(cudaGetLastError());
        h->launches += 2;
        return read(h->gm_s, out, 1);
    }
    // z <- (I - 2 w w^T) z with the inner product kept on the device (krylov.h:48-56: alpha = <w, z>; alpha *= -2)
    int reflect(const double *w, double *z)
    {
        RET(h->dot_to(w, z, n, h->gm_s));
        return h->axpy_ratio(z, w, h->gm_s, h->gm_s + 3, -2.0, n);       // gm_s[3] == 1.0
    }
    int make_w(double *w, const double *v, long long k1, double alpha)
    {
        hh_make_w_kernel<<<grid(), 256, 0, s>>>(w, v, k1, alpha, n);
        CK(cudaGetLastError());
        h->launches++;
        double nn = 0.0;
        RET(dot(w, w, &nn));
        div_kernel<<<grid(), 256, 0, s>>>(w, std::sqrt(nn), n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    }
};

// LAPACK dlartg (what scipy's get_lapack_funcs(['lartg']) calls): c, s, r with [c s; -s c] [f; g] = [r; 0]
void lartg(double f, double g, double *c, double *sn, double *r)
{
    if (g == 0.0) { *c = 1.0; *sn = 0.0; *r = f; return; }
    if (f == 0.0) { *c = 0.0; *sn = std::copysign(1.0, g); *r = std::fabs(g); return; }
    const double d = std::sqrt(f * f + g * g);
    *c = std::fabs(f) / d;
    *r = std::copysign(d, f);
    *sn = g / *r;
}

// AMGB_FLAG_MGS selects modified Gram-Schmidt GMRES, which is left-preconditioned; AMGB_FLAG_REORTH is its option
int check_gmres_flags(int32_t flags)
{
    if ((flags & AMGB_FLAG_MGS) && (flags & AMGB_FLAG_FLEXIBLE))
        return fail(AMGB_EINVAL, "gmres: AMGB_FLAG_MGS and AMGB_FLAG_FLEXIBLE exclude each other");
    if ((flags & AMGB_FLAG_REORTH) && !(flags & AMGB_FLAG_MGS))
        return fail(AMGB_EINVAL, "gmres: AMGB_FLAG_REORTH needs AMGB_FLAG_MGS");
    return AMGB_OK;
}
}  // namespace

// ------------------------------------------------------------------------------------------
// GPU-resident modified Gram-Schmidt GMRES: amgb_solve_gmres with AMGB_FLAG_MGS, ml.solve(accel='gmres_mgs').
// Restates pyamg/krylov/_gmres_mgs.py:42-342 (LEFT preconditioning, stop on the preconditioned residual against
// ||M b||, Givens rotations from lartg) with M = one multigrid cycle from a zero guess.  MGS needs only inner
// products, axpys, A and M, so the basis V (gm_W), r and x stay in the level-0 numbering; x goes back to the caller's
// numbering once, at the end.
// Inner iteration j: v = M A V_j is the cycle's iterate L0.x; j + 2 fused MGS steps (mgs_step_kernel, each followed
// by reduce_partials_kernel) are enqueued back to back, every step reading the coefficient the previous reduction
// left in device memory, and mgs_scale_kernel writes V_{j+1} = v * (1 / ||v||).  The host reads the new H column
// (j + 1 coefficients, ||v||^2 before and after the projections) in one copy; with reorth the second MGS pass (and
// then the scaling) is enqueued only after that read shows the reference's test is met.  Givens rotations and the
// back substitution run on the host, as for Householder GMRES.
// ------------------------------------------------------------------------------------------
namespace {
// device scratch of the MGS drivers for K columns: two sets of max_inner + 3 coefficient slots (the MGS pass, the
// reorth pass), then sumsq_blocks() x K partials of ||v||^2 (the first step forms them beside those of <V_0, v>)
int gmres_mgs_scratch(amgb_hierarchy *h, int mi, int K)
{
    const long long count = (2LL * (mi + 3) + kSumsqBlocks) * K;
    if (h->gm_mgs_count >= count) return AMGB_OK;
    if (h->gm_mgs != nullptr) {
        CK(cudaStreamSynchronize(h->stream));            // nothing in flight may still use the buffer being replaced
        h->dfree(h->gm_mgs);
        h->dev_bytes -= (long long)((sizeof(double) * (size_t)h->gm_mgs_count + 255) & ~(size_t)255);
        h->gm_mgs_count = 0;
    }
    RET(h->dalloc(&h->gm_mgs, count));
    h->gm_mgs_count = count;
    return AMGB_OK;
}

int gmres_mgs(Gmres &G, CallerIo &io, const double *b_host, double *x_host, double tol, long long max_outer, int mi,
              bool reorth, bool x0_zero, double *residuals, int32_t max_residuals, int32_t *n_residuals, int32_t *info)
{
    amgb_hierarchy *h = G.h;
    Level &L0 = G.L0;
    const long long n = G.n;
    cudaStream_t s = G.s;
    RET(gmres_mgs_scratch(h, mi, 1));
    double *coef = h->gm_mgs, *coef2 = h->gm_mgs + (mi + 3), *sq_parts = h->gm_mgs + 2 * (mi + 3);
    double *xk = h->gm_lvl[0], *bk = h->gm_lvl[1], *upd = h->gm_lvl[2];
    const size_t vbytes = sizeof(double) * (size_t)n;
    const int nb = sumsq_blocks(h->S);
    RET(load_level0(h, b_host, x0_zero ? nullptr : x_host, io.in_kind()));
    CK(cudaMemcpyAsync(bk, L0.b, vbytes, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(xk, L0.x, vbytes, cudaMemcpyDeviceToDevice, s));

    // ||M b|| before r: a cycle from zero depends on its rhs alone, so the order changes no value, and r, computed
    // last, is still in L0.x for the first basis vector
    double t = 0.0, normMb = 1.0;                                            // :204-207
    RET(G.dot(bk, bk, &t));
    if (t != 0.0) {
        RET(h->copy_vec(L0.b, bk, n));
        RET(G.precond());
        RET(G.dot(L0.x, L0.x, &t));
        normMb = std::sqrt(t);
    }
    auto residual = [&]() -> int {                                           // L0.x = M (b - A x)   (:192-195)
        RET(h->spmv(OP_RESID, L0.A, xk, bk, L0.b));
        return G.precond();
    };
    RET(residual());
    RET(G.dot(L0.x, L0.x, &t));
    double normr = std::sqrt(t);
    std::vector<double> res{normr};                                          // :197-198
    int status = -2, niter = 0;
    if (normr < tol * normMb) status = 0;                                    // :209-210

    // one MGS pass over v = L0.x against V_0 .. V_inner: coefficients -> c[0 .. inner]; with `norms` also ||v||^2
    // before (first step, normv_old) -> c[inner + 1] and after (last step, normv) -> c[inner + 2]
    auto mgs_pass = [&](int inner, double *c, bool norms) -> int {
        for (int k = 0; k <= inner + 1; k++) {
            const bool last = k == inner + 1, sq = norms && (k == 0 || last);
            mgs_step_kernel<<<nb, 256, 0, s>>>(L0.x, k > 0 ? G.W(k - 1) : nullptr, c + (k > 0 ? k - 1 : 0),
                                               last ? nullptr : G.W(k), n, last ? nullptr : h->sumsq_parts,
                                               sq ? sq_parts : nullptr);
            CK(cudaGetLastError());
            h->launches++;
            if (!last) {
                reduce_partials_kernel<<<1, 1024, 0, s>>>(h->sumsq_parts, nb, c + k);
                CK(cudaGetLastError());
                h->launches++;
            }
            if (sq) {
                reduce_partials_kernel<<<1, 1024, 0, s>>>(sq_parts, nb, c + inner + (last ? 2 : 1));
                CK(cudaGetLastError());
                h->launches++;
            }
        }
        return AMGB_OK;
    };
    auto scale_next = [&](int inner) -> int {                                // V[inner+1] = v / normv (:268-269)
        mgs_scale_kernel<<<G.grid(), 256, 0, s>>>(G.W(inner + 1), L0.x, coef + inner + 2, n);
        CK(cudaGetLastError());
        h->launches++;
        return AMGB_OK;
    };
    std::vector<double> H((size_t)mi * mi), Q((size_t)4 * mi), g((size_t)mi + 1), hv((size_t)mi + 2), y((size_t)mi);
    double *col = nullptr;                                                   // one H column as read from the device
    CK(cudaHostAlloc((void **)&col, sizeof(double) * ((size_t)mi + 3), cudaHostAllocDefault));
    struct PinGuard { double *p; ~PinGuard() { if (p) cudaFreeHost(p); } } pin_guard{col};

    for (long long outer = 0; outer < max_outer && status == -2; outer++) {
        RET(h->scale_to(G.W(0), 1.0 / normr, L0.x, n));                     // V[0] = r * (1 / normr) (:225-226)
        std::fill(H.begin(), H.end(), 0.0);
        std::fill(Q.begin(), Q.end(), 0.0);
        std::fill(g.begin(), g.end(), 0.0);
        g[0] = normr;                                                        // :230-231
        int inner = 0;
        for (inner = 0; inner < mi; inner++) {
            RET(h->spmv(OP_SPMV, L0.A, G.W(inner), nullptr, L0.b));         // v = M (A V[inner])  (:237)
            RET(G.precond());
            RET(mgs_pass(inner, coef, true));                                // :238-258
            if (!reorth) RET(scale_next(inner));
            CK(cudaMemcpyAsync(col, coef, sizeof(double) * ((size_t)inner + 3), cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            for (int k = 0; k <= inner; k++) hv[(size_t)k] = col[k];
            const double normv_old = std::sqrt(col[inner + 1]), normv = std::sqrt(col[inner + 2]);
            hv[(size_t)inner + 1] = normv;                                   // H[inner, inner+1] (:257)
            if (reorth && normv_old == normv_old + 0.001 * normv) {          // :260-266 (normv is not recomputed)
                RET(mgs_pass(inner, coef2, false));
                CK(cudaMemcpyAsync(col, coef2, sizeof(double) * ((size_t)inner + 1), cudaMemcpyDeviceToHost, s));
                CK(cudaStreamSynchronize(s));
                for (int k = 0; k <= inner; k++) hv[(size_t)k] = hv[(size_t)k] + col[k];
            }
            if (reorth) RET(scale_next(inner));
            for (int rot = 0; rot < inner; rot++) {                          // apply_givens (:13-39, :272-273)
                const double xt = hv[(size_t)rot];
                hv[(size_t)rot] = Q[(size_t)4 * rot] * xt + Q[(size_t)4 * rot + 1] * hv[(size_t)rot + 1];
                hv[(size_t)rot + 1] = Q[(size_t)4 * rot + 2] * xt + Q[(size_t)4 * rot + 3] * hv[(size_t)rot + 1];
            }
            if (inner != n - 1 && hv[(size_t)inner + 1] != 0.0) {            // :278-290
                double c, sn, rr;
                lartg(hv[(size_t)inner], hv[(size_t)inner + 1], &c, &sn, &rr);
                double *q = &Q[(size_t)4 * inner];
                q[0] = c; q[1] = sn; q[2] = -sn; q[3] = c;
                const double g0 = g[(size_t)inner], g1 = g[(size_t)inner + 1];
                g[(size_t)inner] = c * g0 + sn * g1;
                g[(size_t)inner + 1] = -sn * g0 + c * g1;
                hv[(size_t)inner] = c * hv[(size_t)inner] + sn * hv[(size_t)inner + 1];
                hv[(size_t)inner + 1] = 0.0;
            }
            for (int k = 0; k < mi; k++) H[(size_t)k * mi + inner] = hv[(size_t)k];   // H[inner, :] (transposed)
            niter++;                                                         // :292
            if (inner < mi - 1) {                                            // :296-302
                normr = std::fabs(g[(size_t)inner + 1]);
                if (normr < tol * normMb) break;
                res.push_back(normr);
            }
        }
        if (inner == mi) inner = mi - 1;                                     // Python's loop variable after a full loop
        const int k = inner + 1;
        for (int i = k - 1; i >= 0; i--) {                                   // solve H[0:k,0:k].T y = g[0:k] (:312)
            double acc = g[(size_t)i];
            for (int j = i + 1; j < k; j++) acc -= H[(size_t)i * mi + j] * y[(size_t)j];
            y[(size_t)i] = acc / H[(size_t)i * mi + i];
        }
        RET(h->scale_to(upd, y[0], G.W(0), n));                              // update = V[:k].T y (:313)
        for (int j = 1; j < k; j++) RET(h->axpby(y[(size_t)j], G.W(j), 1.0, upd, n));
        RET(h->axpby(1.0, upd, 1.0, xk, n));                                 // x = x + update (:314)
        RET(residual());                                                     // :315-319
        RET(G.dot(L0.x, L0.x, &t));
        normr = std::sqrt(t);
        res.push_back(normr);                                                // :324-325
        maxratio_partials_kernel<<<nb, 256, 0, s>>>(upd, xk, n, h->sumsq_parts);   // :328-334
        CK(cudaGetLastError());
        reduce_max_kernel<<<1, 1024, 0, s>>>(h->sumsq_parts, nb, h->gm_s + 1);
        CK(cudaGetLastError());
        h->launches += 2;
        double change = 0.0;
        RET(G.read(h->gm_s + 1, &change, 1));
        if (change >= 0.0 && change < 1e-12) { status = -1; break; }
        if (normr < tol * normMb) { status = 0; break; }                    // :337-338
    }
    if (status == -2) status = niter;                                        // :342
    CK(cudaMemcpyAsync(L0.x_home, xk, vbytes, cudaMemcpyDeviceToDevice, s));
    L0.x = L0.x_home;
    RET(store_level0(h, x_host, io.out_kind()));
    RET(io.end());
    if (!io.dev) CK(cudaStreamSynchronize(s));
    const int nres = (int)std::min<size_t>(res.size(), (size_t)std::max(max_residuals, 0));
    if (residuals != nullptr)
        for (int k = 0; k < nres; k++) residuals[k] = res[(size_t)k];
    if (n_residuals != nullptr) *n_residuals = (int32_t)res.size();
    if (info != nullptr) *info = status;
    h->last_launches = h->launches;
    return AMGB_OK;
}
}  // namespace

extern "C" int amgb_solve_gmres(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t restart,
                                int32_t maxiter, int32_t cycle, int32_t flags, double *residuals,
                                int32_t max_residuals, int32_t *n_residuals, int32_t *info)
{
    RET(check_cycle_args(h, cycle, 1));
    if (b_host == nullptr || x_host == nullptr) return fail(AMGB_EINVAL, "null host vector");
    if (restart < 0) return fail(AMGB_EINVAL, "restart < 0");
    RET(check_gmres_flags(flags));
    CK(cudaSetDevice(h->device));
    Gmres G(h, cycle);
    const long long n = G.n;
    if (n < 2) return fail(AMGB_EINVAL, "gmres: n < 2 is the caller's closed form (b / A[0,0])");
    CallerIo io(h, flags);
    RET(io.begin(b_host, x_host));
    const bool flex = (flags & AMGB_FLAG_FLEXIBLE) != 0;
    // _gmres_householder.py:129-149
    long long max_outer, max_inner;
    if (restart > 0) {
        max_outer = maxiter > 0 ? maxiter : 1;
        max_inner = std::min<long long>(restart, n);
    } else {
        max_outer = 1;
        max_inner = maxiter > 0 ? std::min<long long>(maxiter, n) : std::min<long long>(n, 40);
    }
    const int mi = (int)max_inner;
    cudaStream_t s = h->stream;
    h->launches = 0;
    if (h->gm_W == nullptr || h->gm_inner < mi || (flex && !h->gm_flex)) {
        CK(cudaStreamSynchronize(s));                    // nothing in flight may still use the buffers being replaced
        h->dfree(h->gm_W);
        h->dfree(h->gm_Z);
        RET(h->dalloc(&h->gm_W, (long long)(mi + 1) * G.npad));
        if (flex || h->gm_flex) RET(h->dalloc(&h->gm_Z, (long long)mi * G.npad));
        if (h->gm_s == nullptr) {
            for (int k = 0; k < 4; k++) RET(h->dalloc(&h->gm_vec[k], G.npad));
            for (int k = 0; k < 3; k++) RET(h->dalloc(&h->gm_lvl[k], G.npad));
            RET(h->dalloc(&h->gm_s, 8));
            const double init[4] = {0.0, 0.0, 0.0, 1.0};
            CK(cudaMemcpy(h->gm_s, init, sizeof init, cudaMemcpyHostToDevice));
        }
        h->gm_inner = mi;
        h->gm_flex = h->gm_flex || flex;
    }
    if (cycle == AMGB_CYCLE_AMLI) RET(h->prepare_amli());
    if (flags & AMGB_FLAG_MGS)
        return gmres_mgs(G, io, b_host, x_host, tol, max_outer, mi, (flags & AMGB_FLAG_REORTH) != 0,
                         (flags & AMGB_FLAG_X0_ZERO) != 0, residuals, max_residuals, n_residuals, info);
    double *v = h->gm_vec[0], *xk = h->gm_vec[1], *bk = h->gm_vec[2], *upd = h->gm_vec[3];
    double *b_lvl = h->gm_lvl[0], *lin = h->gm_lvl[1], *lout = h->gm_lvl[2];
    Level &L0 = G.L0;
    const size_t vbytes = sizeof(double) * (size_t)n;
    CK(cudaMemcpyAsync(bk, b_host, vbytes, io.in_kind(), s));
    if (flags & AMGB_FLAG_X0_ZERO) RET(h->launch_count_fill(xk, n));
    else CK(cudaMemcpyAsync(xk, x_host, vbytes, io.in_kind(), s));
    RET(G.to_level(bk, b_lvl));

    // r = b - A x (then r = M r for the left-preconditioned method) -> the first reflector's storage W(0)
    auto residual_to_w0 = [&]() -> int {
        RET(G.to_level(xk, lin));
        if (flex) {
            RET(h->spmv(OP_RESID, L0.A, lin, b_lvl, lout));
            return G.from_level(lout, G.W(0));
        }
        RET(h->spmv(OP_RESID, L0.A, lin, b_lvl, L0.b));
        RET(G.precond());
        return G.from_level(L0.x, G.W(0));
    };
    std::vector<double> res;
    double t = 0.0, normr = 0.0;
    RET(residual_to_w0());
    RET(G.dot(G.W(0), G.W(0), &t));
    normr = std::sqrt(t);
    res.push_back(normr);                                                   // :165-167
    double scale = 1.0;                                                     // :169-174 / _fgmres.py:171-174
    RET(G.dot(bk, bk, &t));
    if (t != 0.0) {
        if (flex) {
            scale = std::sqrt(t);
        } else {
            RET(h->copy_vec(L0.b, b_lvl, n));
            RET(G.precond());
            RET(G.from_level(L0.x, v));
            RET(G.dot(v, v, &t));
            scale = std::sqrt(t);
        }
    }
    int status = -2, niter = 0;
    if (normr < tol * scale) status = 0;                                    // :177-178
    const int m2 = (int)std::min<long long>(n, (long long)mi + 1);          // leading entries of v the host needs
    std::vector<double> H((size_t)mi * mi), Q((size_t)4 * mi), g((size_t)mi + 1), hv((size_t)m2), y((size_t)mi);
    double *hv_pinned = nullptr;
    CK(cudaHostAlloc((void **)&hv_pinned, sizeof(double) * (size_t)m2, cudaHostAllocDefault));
    struct PinGuard { double *p; ~PinGuard() { if (p) cudaFreeHost(p); } } pin_guard{hv_pinned};

    for (long long outer = 0; outer < max_outer && status == -2; outer++) {
        // first reflector from r: w = r; w[0] += sign(r[0]) ||r||; w /= ||w||          (:186-192)
        double r0 = 0.0;
        RET(G.read(G.W(0), &r0, 1));
        const double beta = (r0 == 0.0 ? 1.0 : r0 / std::fabs(r0)) * normr;
        RET(G.make_w(G.W(0), G.W(0), 0, beta));
        CK(cudaMemsetAsync(G.W(1), 0, sizeof(double) * (size_t)mi * (size_t)G.npad, s));   // W = zeros (:203)
        std::fill(H.begin(), H.end(), 0.0);
        std::fill(Q.begin(), Q.end(), 0.0);
        std::fill(g.begin(), g.end(), 0.0);
        g[0] = -beta;                                                        // :208-209
        int inner = 0;
        for (inner = 0; inner < mi; inner++) {
            hh_unit_reflect_kernel<<<G.grid(), 256, 0, s>>>(v, G.W(inner), inner, n);      // :214-215
            CK(cudaGetLastError());
            h->launches++;
            for (int j = inner - 1; j >= 0; j--) RET(G.reflect(G.W(j), v));                 // :219
            if (flex) {                                                      // _fgmres.py:221-230
                RET(G.to_level(v, L0.b));
                RET(G.precond());
                RET(G.from_level(L0.x, G.Z(inner)));
                RET(h->spmv(OP_SPMV, L0.A, L0.x, nullptr, lout));
                RET(G.from_level(lout, v));
            } else {                                                         // :222-225
                RET(G.to_level(v, lin));
                RET(h->spmv(OP_SPMV, L0.A, lin, nullptr, L0.b));
                RET(G.precond());
                RET(G.from_level(L0.x, v));
            }
            for (int j = 0; j <= inner; j++) RET(G.reflect(G.W(j), v));                     // :235
            CK(cudaMemcpyAsync(hv_pinned, v, sizeof(double) * (size_t)m2, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            for (int k = 0; k < m2; k++) hv[(size_t)k] = hv_pinned[k];
            if (inner != n - 1) {                                            // :244-263
                double alpha = 0.0;
                RET(G.sumsq_from(v, inner + 1, &alpha));
                alpha = std::sqrt(alpha);
                if (alpha != 0.0) {
                    const double v0 = hv[(size_t)inner + 1];
                    alpha = (v0 == 0.0 ? 1.0 : v0 / std::fabs(v0)) * alpha;
                    if (inner < mi - 1) RET(G.make_w(G.W(inner + 1), v, inner + 1, alpha));
                    hv[(size_t)inner + 1] = -alpha;
                    for (int k = inner + 2; k < m2; k++) hv[(size_t)k] = 0.0;
                }
            }
            for (int rot = 0; rot < inner; rot++) {                          // apply_givens (krylov.h:171-186)
                const double xt = hv[(size_t)rot];
                hv[(size_t)rot] = Q[(size_t)4 * rot] * xt + Q[(size_t)4 * rot + 1] * hv[(size_t)rot + 1];
                hv[(size_t)rot + 1] = Q[(size_t)4 * rot + 2] * xt + Q[(size_t)4 * rot + 3] * hv[(size_t)rot + 1];
            }
            if (inner != n - 1 && hv[(size_t)inner + 1] != 0.0) {            // :276-291
                double c, sn, rr;
                lartg(hv[(size_t)inner], hv[(size_t)inner + 1], &c, &sn, &rr);
                double *q = &Q[(size_t)4 * inner];
                q[0] = c; q[1] = sn; q[2] = -sn; q[3] = c;
                const double g0 = g[(size_t)inner], g1 = g[(size_t)inner + 1];
                g[(size_t)inner] = c * g0 + sn * g1;
                g[(size_t)inner + 1] = -sn * g0 + c * g1;
                hv[(size_t)inner] = c * hv[(size_t)inner] + sn * hv[(size_t)inner + 1];
                hv[(size_t)inner + 1] = 0.0;
            }
            for (int k = 0; k < mi; k++) H[(size_t)k * mi + inner] = hv[(size_t)k];         // H[:, inner] (:295)
            if (!flex) niter++;                                              // :297
            if (inner < mi - 1) {                                            // :301-305
                normr = std::fabs(g[(size_t)inner + 1]);
                if (normr < tol * scale) break;                              // (fgmres: before niter += 1)
                res.push_back(normr);
            }
            if (flex) niter++;                                               // _fgmres.py:306
        }
        if (inner == mi) inner = mi - 1;                                     // Python's loop variable after a full loop
        const int k = inner + 1;
        for (int i = k - 1; i >= 0; i--) {                                   // solve H[0:k,0:k] y = g[0:k] (upper triangular)
            double acc = g[(size_t)i];
            for (int j = i + 1; j < k; j++) acc -= H[(size_t)i * mi + j] * y[(size_t)j];
            y[(size_t)i] = acc / H[(size_t)i * mi + i];
        }
        if (flex) {                                                          // update = Z[:, 0:k] y (_fgmres.py:321)
            RET(h->scale_to(upd, y[0], G.Z(0), n));
            for (int j = 1; j < k; j++) RET(h->axpby(y[(size_t)j], G.Z(j), 1.0, upd, n));
        } else {                                                             // householder_hornerscheme (:321-322)
            RET(h->launch_count_fill(upd, n));
            for (int j = k - 1; j >= 0; j--) {
                add_at_kernel<<<1, 1, 0, s>>>(upd, j, y[(size_t)j]);
                CK(cudaGetLastError());
                h->launches++;
                RET(G.reflect(G.W(j), upd));
            }
        }
        RET(h->axpby(1.0, upd, 1.0, xk, n));                                 // x = x + update (:324)
        RET(residual_to_w0());                                               // :325-328
        RET(G.dot(G.W(0), G.W(0), &t));
        normr = std::sqrt(t);
        res.push_back(normr);                                                // :335-336
        maxratio_partials_kernel<<<sumsq_blocks(h->S), 256, 0, s>>>(upd, xk, n, h->sumsq_parts);   // :339-346
        CK(cudaGetLastError());
        reduce_max_kernel<<<1, 1024, 0, s>>>(h->sumsq_parts, sumsq_blocks(h->S), h->gm_s + 1);
        CK(cudaGetLastError());
        h->launches += 2;
        double change = 0.0;
        RET(G.read(h->gm_s + 1, &change, 1));
        if (change >= 0.0 && change < 1e-12) { status = -1; break; }
        if (normr < tol * scale) { status = 0; break; }                     // :349-350
    }
    if (status == -2) status = niter;                                        // :354
    CK(cudaMemcpyAsync(x_host, xk, vbytes, io.out_kind(), s));
    RET(io.end());
    if (!io.dev) CK(cudaStreamSynchronize(s));
    L0.x = L0.x_home;
    const int nres = (int)std::min<size_t>(res.size(), (size_t)std::max(max_residuals, 0));
    if (residuals != nullptr)
        for (int k = 0; k < nres; k++) residuals[k] = res[(size_t)k];
    if (n_residuals != nullptr) *n_residuals = (int32_t)res.size();
    if (info != nullptr) *info = status;
    h->last_launches = h->launches;
    return AMGB_OK;
}

// ------------------------------------------------------------------------------------------
// GPU-resident right-preconditioned BiCGStab: ml.solve(accel='bicgstab') with every vector in HBM.
// Restates pyamg/krylov/_bicgstab.py:10-200 (criteria 'rr') with M = one multigrid cycle from x0 = 0.  Like CG the
// method is invariant under the level-0 row permutation, so all vectors live in the level numbering; the
// preconditioned directions M p and M s are read straight out of the cycle's iterate buffer.
// ------------------------------------------------------------------------------------------
extern "C" int amgb_solve_bicgstab(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t maxiter,
                                   int32_t cycle, int32_t flags, double *residuals, int32_t *n_residuals, int32_t *info)
{
    RET(check_cycle_args(h, cycle, 1));
    if (b_host == nullptr || x_host == nullptr) return fail(AMGB_EINVAL, "null host vector");
    if (maxiter < 1) return fail(AMGB_EINVAL, "Number of iterations must be positive");    // _bicgstab.py:92-93
    CK(cudaSetDevice(h->device));
    Level &L0 = h->levels[0];
    const long long n = L0.A.n_rows;
    if (n < 2) return fail(AMGB_EINVAL, "bicgstab: n < 2 is the caller's closed form (b / A[0,0])");
    CallerIo io(h, flags);
    RET(io.begin(b_host, x_host));
    cudaStream_t s = h->stream;
    h->launches = 0;
    if (h->kry[0] == nullptr)
        for (int k = 0; k < 4; k++) RET(h->dalloc(&h->kry[k], n + 2));
    if (h->kry2[0] == nullptr)
        for (int k = 0; k < 4; k++) RET(h->dalloc(&h->kry2[k], n + 2));
    double *xk = h->kry[0], *p = h->kry[1], *AMp = h->kry[2], *bk = h->kry[3];
    double *r = h->kry2[0], *rstar = h->kry2[1], *sv = h->kry2[2], *AMs = h->kry2[3];
    const size_t vbytes = sizeof(double) * (size_t)n;
    RET(load_level0(h, b_host, (flags & AMGB_FLAG_X0_ZERO) ? nullptr : x_host, io.in_kind()));
    CK(cudaMemcpyAsync(bk, L0.b, vbytes, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(xk, L0.x, vbytes, cudaMemcpyDeviceToDevice, s));
    auto precond_of = [&](const double *v) -> int {        // L0.x <- M v
        CK(cudaMemcpyAsync(L0.b, v, vbytes, cudaMemcpyDeviceToDevice, s));
        L0.x = L0.x_home;
        RET(h->launch_count_fill(L0.x, n));
        return h->one_iteration(cycle, 1);
    };
    double t = 0, rrstar_old = 0, rrstar_new = 0, d1 = 0, d2 = 0;
    RET(h->spmv(OP_RESID, L0.A, xk, bk, r));                          // r = b - A x             (:96)
    RET(dev_dot(h, r, r, n, &t));
    std::vector<double> res;
    res.push_back(std::sqrt(t));                                      // :97-100
    RET(dev_dot(h, bk, bk, n, &t));
    double normb = std::sqrt(t);
    if (normb == 0.0) normb = 1.0;                                    // :103-106
    const double rtol = tol * normb;                                  // criteria 'rr' (:109-110)
    int it = 0, status = -2;
    if (res.back() < rtol) status = 0;                                // :122-123
    if (status == -2) {
        CK(cudaMemcpyAsync(rstar, r, vbytes, cudaMemcpyDeviceToDevice, s));   // :131-132
        CK(cudaMemcpyAsync(p, r, vbytes, cudaMemcpyDeviceToDevice, s));
        RET(dev_dot(h, rstar, r, n, &rrstar_old));                    // :134
    }
    while (status == -2) {
        RET(precond_of(p));                                           // Mp = M p                (:140)
        RET(h->spmv(OP_SPMV, L0.A, L0.x, nullptr, AMp));              // AMp = A Mp              (:141)
        RET(dev_dot(h, rstar, AMp, n, &d1));
        const double alpha = rrstar_old / d1;                         // :144
        RET(dev_axpby(h, alpha, L0.x, 1.0, xk, n));                   // x += alpha Mp           (:155, first term)
        CK(cudaMemcpyAsync(sv, r, vbytes, cudaMemcpyDeviceToDevice, s));
        RET(dev_axpby(h, -alpha, AMp, 1.0, sv, n));                   // s = r - alpha AMp       (:147)
        RET(precond_of(sv));                                          // Ms = M s                (:148)
        RET(h->spmv(OP_SPMV, L0.A, L0.x, nullptr, AMs));              // AMs = A Ms              (:149)
        RET(dev_dot(h, AMs, sv, n, &d1));
        RET(dev_dot(h, AMs, AMs, n, &d2));
        const double omega = d1 / d2;                                 // :152
        RET(dev_axpby(h, omega, L0.x, 1.0, xk, n));                   // x += omega Ms           (:155, second term)
        CK(cudaMemcpyAsync(r, sv, vbytes, cudaMemcpyDeviceToDevice, s));
        RET(dev_axpby(h, -omega, AMs, 1.0, r, n));                    // r = s - omega AMs       (:158)
        RET(dev_dot(h, rstar, r, n, &rrstar_new));                    // :161
        const double beta = (rrstar_new / rrstar_old) * (alpha / omega);      // :162
        rrstar_old = rrstar_new;
        RET(dev_axpby(h, -omega, AMp, 1.0, p, n));                    // p - omega AMp
        RET(dev_axpby(h, 1.0, r, beta, p, n));                        // p = r + beta (p - omega AMp)   (:166)
        it++;
        RET(dev_dot(h, r, r, n, &t));
        res.push_back(std::sqrt(t));                                  // :170-173
        if (res.back() < rtol) { status = 0; break; }                 // :184-185
        if (it == maxiter) { status = it; break; }                    // :187-188
    }
    CK(cudaMemcpyAsync(L0.x_home, xk, vbytes, cudaMemcpyDeviceToDevice, s));
    L0.x = L0.x_home;
    RET(store_level0(h, x_host, io.out_kind()));
    RET(io.end());
    if (!io.dev) CK(cudaStreamSynchronize(s));
    if (residuals != nullptr)
        for (size_t k = 0; k < res.size() && k < (size_t)maxiter + 1; k++) residuals[k] = res[k];
    if (n_residuals != nullptr) *n_residuals = (int32_t)res.size();
    if (info != nullptr) *info = status;
    h->last_launches = h->launches;
    return AMGB_OK;
}
