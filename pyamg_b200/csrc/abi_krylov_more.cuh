// abi_krylov_more.cuh -- part of engine.cu's translation unit (included there): amgb_hierarchy_set_transpose0 and
// amgb_solve_krylov, the GPU-resident CGNR, CGNE, minimal residual and steepest descent of
// MultilevelSolver.solve(accel='cgnr' | 'cgne' | 'minimal_residual' | 'steepest_descent').
//
// Each driver restates the reference's function (pyamg/krylov/_cgnr.py:97-220, _cgne.py:97-214,
// _minimal_residual.py:92-163, _steepest_descent.py:92-197; criteria 'rr') with M = one multigrid cycle from a zero
// guess (aspreconditioner), in the manner of amgb_solve_cg: every vector in level-0 numbering, the preconditioner's
// right-hand side in L0.b and its result in L0.x, dot products through dev_dot (fixed grid, two stages), updates
// through axpby_kernel, SpMVs and residuals through h->spmv.  The host reads scalars only.
#pragma once

static void free_dev_csr(amgb_hierarchy *h, DevCsr &D)
{
    h->dfree(D.Ap); h->dfree(D.Aj); h->dfree(D.Ax); h->dfree(D.tiles);
    h->dfree(D.codes); h->dfree(D.dict); h->dfree(D.pairs); h->dfree(D.rcodes); h->dfree(D.patterns);
    D = DevCsr();
}

// A^H of the fine level (the caller's A.T.conjugate().tocsr(): row i holds column i of A, in ascending row order of
// A, the order SciPy's csc_matvec sums A^H r in), permuted like level 0.  Replaces an earlier one.
extern "C" int amgb_hierarchy_set_transpose0(amgb_hierarchy *h, const amgb_matrix *AH)
{
    if (h == nullptr) return fail(AMGB_EINVAL, "null hierarchy");
    if (!h->finalized) return fail(AMGB_ESTATE, "hierarchy not finalized");
    HostCsr H;
    RET(to_host_csr(AH, H, "AH"));
    const long long n = h->levels[0].A.n_rows;
    if (H.n_rows != n || H.n_cols != n) return fail(AMGB_EINVAL, "AH: shape differs from the fine-level operator");
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));              // no solve in flight may still read the one being replaced
    free_dev_csr(h, h->At0);
    if (h->order0 == nullptr) return h->upload_csr(H, h->At0);
    std::vector<int> order((size_t)n), pos((size_t)n);
    CK(cudaMemcpy(order.data(), h->order0, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(pos.data(), h->pos0, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost));
    HostCsr T;
    permute_csr(H, order.data(), pos.data(), T);
    return h->upload_csr(T, h->At0);
}

extern "C" int amgb_solve_krylov(amgb_hierarchy *h, int32_t method, const double *b_host, double *x_host, double tol,
                                 int32_t maxiter, int32_t cycle, int32_t flags, double *residuals,
                                 int32_t *n_residuals, int32_t *info, int32_t *reason)
{
    RET(check_cycle_args(h, cycle, 1));
    if (method < AMGB_KRYLOV_CGNR || method > AMGB_KRYLOV_SD) return fail(AMGB_EINVAL, "unknown Krylov method");
    if (b_host == nullptr || x_host == nullptr) return fail(AMGB_EINVAL, "null host vector");
    if (maxiter < 1) return fail(AMGB_EINVAL, "Number of iterations must be positive");
    const bool normal = method == AMGB_KRYLOV_CGNR || method == AMGB_KRYLOV_CGNE;
    if (normal && h->At0.Ap == nullptr) return fail(AMGB_ESTATE, "CGNR / CGNE: amgb_hierarchy_set_transpose0 first");
    CK(cudaSetDevice(h->device));
    CallerIo io(h, flags);
    RET(io.begin(b_host, x_host));
    Level &L0 = h->levels[0];
    const long long n = L0.A.n_rows;
    const size_t vbytes = sizeof(double) * (size_t)n;
    cudaStream_t s = h->stream;
    h->launches = 0;
    if (h->kry[0] == nullptr)
        for (int k = 0; k < 4; k++) RET(h->dalloc(&h->kry[k], n + 2));
    if (h->kry2[0] == nullptr)
        for (int k = 0; k < 4; k++) RET(h->dalloc(&h->kry2[k], n + 2));
    double *xk = h->kry[0], *bk = h->kry[3], *u = h->kry[1], *v = h->kry[2], *w = h->kry2[0];
    RET(load_level0(h, b_host, (flags & AMGB_FLAG_X0_ZERO) ? nullptr : x_host, io.in_kind()));
    CK(cudaMemcpyAsync(bk, L0.b, vbytes, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(xk, L0.x, vbytes, cudaMemcpyDeviceToDevice, s));
    auto precond = [&]() -> int {                         // L0.x = M L0.b: one cycle from zero
        L0.x = L0.x_home;
        RET(h->launch_count_fill(L0.x, n));
        return h->one_iteration(cycle, 1);
    };
    double t = 0.0;
    RET(dev_dot(h, bk, bk, n, &t));
    const double normb0 = std::sqrt(t);
    std::vector<double> res;
    int it = 0, status = -2, why = AMGB_REASON_NONE;

    if (method == AMGB_KRYLOV_CGNR) {
        // r = w, rhat = L0.b, z = L0.x, p = u, A p = v
        double *r = w, *p = u, *Ap = v;
        const double rtol = tol * (normb0 == 0.0 ? 1.0 : normb0);                  // :131-138
        RET(h->spmv(OP_RESID, L0.A, xk, bk, r));                                   // r = b - A x        (:119)
        RET(h->spmv(OP_SPMV, h->At0, r, nullptr, L0.b));                          // rhat = A^H r       (:120)
        RET(precond());                                                            // z = M rhat         (:124)
        CK(cudaMemcpyAsync(p, L0.x, vbytes, cudaMemcpyDeviceToDevice, s));         // p = z              (:125)
        double zr = 0.0;
        RET(dev_dot(h, L0.x, L0.b, n, &zr));                                       // <z, rhat>          (:126)
        RET(dev_dot(h, r, r, n, &t));
        res.push_back(std::sqrt(t));                                               // :121, :128-129
        if (res.back() < rtol) status = 0;                                         // :157-158
        while (status == -2) {
            RET(h->spmv(OP_SPMV, L0.A, p, nullptr, Ap));                           // w = A p            (:166)
            RET(dev_dot(h, Ap, Ap, n, &t));
            const double alpha = zr / t;                                           // :169
            RET(dev_axpby(h, alpha, p, 1.0, xk, n));                               // x += alpha p       (:172)
            if ((it % 8) != 0 && it > 0) RET(dev_axpby(h, -alpha, Ap, 1.0, r, n)); // r -= alpha w       (:175-176)
            else RET(h->spmv(OP_RESID, L0.A, xk, bk, r));                          // r = b - A x        (:177-178)
            RET(h->spmv(OP_SPMV, h->At0, r, nullptr, L0.b));                      // rhat = A^H r       (:181)
            RET(precond());                                                        // z = M rhat         (:184)
            double zr_new = 0.0;
            RET(dev_dot(h, L0.x, L0.b, n, &zr_new));                               // :187
            const double beta = zr_new / zr;                                       // :188-189
            zr = zr_new;
            RET(dev_axpby(h, 1.0, L0.x, beta, p, n));                              // p = beta p + z     (:192-193)
            it++;
            RET(dev_dot(h, r, r, n, &t));
            res.push_back(std::sqrt(t));                                           // :196-199
            if (res.back() < rtol) { status = 0; break; }                          // :216-217
            if (it == maxiter) { status = it; break; }                             // :219-220
        }
    } else if (method == AMGB_KRYLOV_CGNE) {
        // r = L0.b, z = L0.x, p = u, A p and A^H z = v
        double *r = L0.b, *p = u, *tmp = v;
        const double rtol = tol * (normb0 == 0.0 ? 1.0 : normb0);                  // :130-137
        RET(h->spmv(OP_RESID, L0.A, xk, bk, r));                                   // r = b - A x        (:119)
        RET(precond());                                                            // z = M r            (:123)
        RET(h->spmv(OP_SPMV, h->At0, L0.x, nullptr, p));                          // p = A^H z          (:124)
        double zr = 0.0;
        RET(dev_dot(h, L0.x, r, n, &zr));                                          // <z, r>             (:125)
        RET(dev_dot(h, r, r, n, &t));
        res.push_back(std::sqrt(t));                                               // :120, :127-128
        if (res.back() < rtol) status = 0;                                         // :156-157
        while (status == -2) {
            RET(dev_dot(h, p, p, n, &t));
            const double alpha = zr / t;                                           // :166
            RET(dev_axpby(h, alpha, p, 1.0, xk, n));                               // x += alpha p       (:169)
            if ((it % 8) != 0 && it > 0) {
                RET(h->spmv(OP_SPMV, L0.A, p, nullptr, tmp));
                RET(dev_axpby(h, -alpha, tmp, 1.0, r, n));                         // r -= alpha A p     (:172-173)
            } else {
                RET(h->spmv(OP_RESID, L0.A, xk, bk, r));                           // r = b - A x        (:174-175)
            }
            RET(precond());                                                        // z = M r            (:178)
            double zr_new = 0.0;
            RET(dev_dot(h, L0.x, r, n, &zr_new));                                  // :181
            const double beta = zr_new / zr;                                       // :182-183
            zr = zr_new;
            RET(h->spmv(OP_SPMV, h->At0, L0.x, nullptr, tmp));
            RET(dev_axpby(h, 1.0, tmp, beta, p, n));                               // p = beta p + A^H z (:186-187)
            it++;
            RET(dev_dot(h, r, r, n, &t));
            res.push_back(std::sqrt(t));                                           // :190-193
            if (res.back() < rtol) { status = 0; break; }                          // :210-211
            if (it == maxiter) { status = it; break; }                             // :213-214
        }
    } else if (method == AMGB_KRYLOV_MR) {
        // r and A z = L0.b, p = L0.x, z = u (a copy: the next cycle overwrites L0.x)
        double *z = u;
        RET(h->spmv(OP_RESID, L0.A, xk, bk, L0.b));                                // r = b - A x        (:107)
        RET(precond());                                                            // z = M r            (:108)
        CK(cudaMemcpyAsync(z, L0.x, vbytes, cudaMemcpyDeviceToDevice, s));
        RET(dev_dot(h, z, z, n, &t));
        res.push_back(std::sqrt(t));                                               // ||z||              (:109-113)
        double normMb = 1.0;                                                       // :116-120
        if (normb0 != 0.0) {
            CK(cudaMemcpyAsync(L0.b, bk, vbytes, cudaMemcpyDeviceToDevice, s));
            RET(precond());
            RET(dev_dot(h, L0.x, L0.x, n, &t));
            normMb = std::sqrt(t);
        }
        const double rtol = tol * normMb;
        if (res.back() < rtol) status = 0;                                         // :123-124
        while (status == -2) {
            RET(h->spmv(OP_SPMV, L0.A, z, nullptr, L0.b));
            RET(precond());                                                        // p = M (A z)        (:132)
            double pz = 0.0;
            RET(dev_dot(h, L0.x, z, n, &pz));                                      // :135
            if (pz < 0.0) { status = -1; why = AMGB_REASON_INDEFINITE_MATRIX; break; }   // :136-138
            RET(dev_dot(h, L0.x, L0.x, n, &t));
            const double alpha = pz / t;                                           // :140
            RET(dev_axpby(h, alpha, z, 1.0, xk, n));                               // x = x + alpha z    (:141)
            it++;
            if ((it % 50) != 0) {                                                  // (sic) :145-147
                RET(h->spmv(OP_RESID, L0.A, xk, bk, L0.b));                        // r = b - A x
                RET(precond());                                                    // z = M r
                CK(cudaMemcpyAsync(z, L0.x, vbytes, cudaMemcpyDeviceToDevice, s));
            } else {
                RET(dev_axpby(h, -alpha, L0.x, 1.0, z, n));                        // z = z - alpha p    (:148-149)
            }
            RET(dev_dot(h, z, z, n, &t));
            res.push_back(std::sqrt(t));                                           // :151-153
            if (res.back() < rtol) { status = 0; break; }                          // :159-160
            if (it == maxiter) { status = it; break; }                             // :162-163
        }
    } else {
        // r = L0.b, z = L0.x, q = u
        double *r = L0.b, *q = u;
        const double rtol = tol * (normb0 == 0.0 ? 1.0 : normb0);                  // :114-120
        RET(h->spmv(OP_RESID, L0.A, xk, bk, r));                                   // r = b - A x        (:104)
        RET(precond());                                                            // z = M r            (:105)
        double rz = 0.0;
        RET(dev_dot(h, r, L0.x, n, &rz));                                          // :106
        RET(dev_dot(h, r, r, n, &t));
        res.push_back(std::sqrt(t));                                               // :108-111 (no test before the loop)
        while (status == -2) {
            RET(h->spmv(OP_SPMV, L0.A, L0.x, nullptr, q));                         // q = A z            (:145)
            double zAz = 0.0;
            RET(dev_dot(h, L0.x, q, n, &zAz));                                     // :146
            if (zAz < 0.0) { status = -1; why = AMGB_REASON_INDEFINITE_MATRIX; break; }  // :147-149
            const double alpha = rz / zAz;                                         // :151
            RET(dev_axpby(h, alpha, L0.x, 1.0, xk, n));                            // x = x + alpha z    (:152)
            it++;
            if ((it % 50) != 0) RET(h->spmv(OP_RESID, L0.A, xk, bk, r));           // (sic) r = b - A x  (:155-156)
            else RET(dev_axpby(h, -alpha, q, 1.0, r, n));                          // r = r - alpha q    (:157-158)
            RET(precond());                                                        // z = M r            (:160)
            RET(dev_dot(h, r, L0.x, n, &rz));                                      // :161
            if (rz < 0.0) { status = -1; why = AMGB_REASON_INDEFINITE_PRECONDITIONER; break; }  // :163-165
            RET(dev_dot(h, r, r, n, &t));
            res.push_back(std::sqrt(t));                                           // :167-170
            if (res.back() < rtol) { status = 0; break; }                          // :187-188
            if (rz == 0.0) { status = -1; why = AMGB_REASON_SINGULAR_PRECONDITIONER; break; }   // :190-194
            if (it == maxiter) { status = it; break; }                             // :196-197
        }
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
    if (reason != nullptr) *reason = why;
    h->last_launches = h->launches;
    return AMGB_OK;
}
