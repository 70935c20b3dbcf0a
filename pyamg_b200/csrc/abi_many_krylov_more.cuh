// abi_many_krylov_more.cuh -- amgb_solve_many_krylov: MultilevelSolver.solve_many(accel='cgnr' | 'cgne' |
// 'minimal_residual' | 'steepest_descent'), the drivers of abi_krylov_more.cuh on up to eight right-hand sides per
// pass over the hierarchy (included by engine.cu after abi_many_krylov.cuh and abi_krylov_more.cuh).
//
// Each group driver restates amgb_solve_krylov line by line, K columns wide, as abi_many_krylov.cuh restates CG and
// BiCGStab: the preconditioner is many_one_iteration, the SpMVs and residuals many_spmv on A and on A^H, the dot
// products many_dot_kernel + many_reduce_kernel and the updates many_axpby_kernel on the active columns.  Column j --
// iterate, residual list, info and reason -- is what amgb_solve_krylov computes on column j, bit for bit.  Scalars,
// status and residual lists live on the host per column; padding columns are inactive from the start.
#pragma once

template <int K>
static int many_more_group(int method, amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X,
                           bool x0_zero, bool dev, double tol, int32_t maxiter, int32_t cycle, double *residuals,
                           int32_t *n_residuals, int32_t *info, int32_t *reason)
{
    RET(many_krylov_prepare<K>(h, 5));
    ManyKrylov<K> M(h, cycle, dev);
    ManyWidth &mw = M.mw;
    const DevCsr &At = h->At0;
    double *xk = mw.kry[0], *u = mw.kry[1], *v = mw.kry[2], *bk = mw.kry[3], *wv = mw.kry[4];
    double *Vb = M.V.b;
    const double *z_out = M.V.x_home;                     // the preconditioner's output
    RET(M.load(B, k, c0, w, bk));
    if (x0_zero) RET(h->launch_count_fill(xk, M.n * K));
    else RET(M.load(X, k, c0, w, xk));
    std::vector<double> normb((size_t)K, 0.0), rtol((size_t)K, 0.0), sc((size_t)K, 0.0), alpha((size_t)K, 0.0);
    std::vector<double> neg_alpha((size_t)K, 0.0), beta((size_t)K, 0.0), ones((size_t)K, 1.0);
    std::vector<std::vector<double>> res((size_t)w);
    std::vector<int> status((size_t)w, -2), why((size_t)w, AMGB_REASON_NONE);
    unsigned act = 0;
    auto on = [&](int q) { return (act & (1u << q)) != 0; };
    auto stop = [&](int q, int st, int r) { status[(size_t)q] = st; why[(size_t)q] = r; act &= ~(1u << q); };
    RET(M.dot(bk, bk, 0));
    RET(M.read(1));
    for (int q = 0; q < w; q++) {
        normb[(size_t)q] = std::sqrt(M.got[(size_t)q]);
        act |= 1u << q;
    }
    int it = 0;

    if (method == AMGB_KRYLOV_CGNR) {
        double *r = wv, *p = u, *Ap = v;
        RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));                 // r = b - A x
        RET(many_spmv<K>(h, OP_SPMV, At, r, nullptr, Vb));               // rhat = A^H r
        RET(M.precond());                                                 // z = M rhat
        RET(M.copy(p, z_out));                                            // p = z
        RET(M.dot(z_out, Vb, 0));
        RET(M.dot(r, r, 1));
        RET(M.read(2));
        for (int q = 0; q < w; q++) {
            sc[(size_t)q] = M.got[(size_t)q];                             // zr
            res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));
            rtol[(size_t)q] = tol * (normb[(size_t)q] == 0.0 ? 1.0 : normb[(size_t)q]);
            if (res[(size_t)q].back() < rtol[(size_t)q]) stop(q, 0, AMGB_REASON_NONE);
        }
        while (act != 0) {
            RET(many_spmv<K>(h, OP_SPMV, M.A0, p, nullptr, Ap));          // w = A p
            RET(M.dot(Ap, Ap, 0));
            RET(M.read(1));
            for (int q = 0; q < w; q++) {
                alpha[(size_t)q] = on(q) ? sc[(size_t)q] / M.got[(size_t)q] : 0.0;
                neg_alpha[(size_t)q] = -alpha[(size_t)q];
            }
            RET(M.axpby(alpha.data(), p, ones.data(), xk, act));          // x += alpha p
            if ((it % 8) != 0 && it > 0) RET(M.axpby(neg_alpha.data(), Ap, ones.data(), r, act));   // r -= alpha w
            else RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));         // r = b - A x
            RET(many_spmv<K>(h, OP_SPMV, At, r, nullptr, Vb));           // rhat = A^H r
            RET(M.precond());                                             // z = M rhat
            RET(M.dot(z_out, Vb, 0));
            RET(M.dot(r, r, 1));
            RET(M.read(2));
            for (int q = 0; q < w; q++) {
                if (!on(q)) continue;
                beta[(size_t)q] = M.got[(size_t)q] / sc[(size_t)q];
                sc[(size_t)q] = M.got[(size_t)q];
            }
            RET(M.axpby(ones.data(), z_out, beta.data(), p, act));        // p = beta p + z
            it++;
            for (int q = 0; q < w; q++) {
                if (!on(q)) continue;
                res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));
                if (res[(size_t)q].back() < rtol[(size_t)q]) stop(q, 0, AMGB_REASON_NONE);
                else if (it == maxiter) stop(q, it, AMGB_REASON_NONE);
            }
        }
    } else if (method == AMGB_KRYLOV_CGNE) {
        double *r = Vb, *p = u, *tmp = v;
        RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));                 // r = b - A x
        RET(M.precond());                                                 // z = M r
        RET(many_spmv<K>(h, OP_SPMV, At, z_out, nullptr, p));            // p = A^H z
        RET(M.dot(z_out, r, 0));
        RET(M.dot(r, r, 1));
        RET(M.read(2));
        for (int q = 0; q < w; q++) {
            sc[(size_t)q] = M.got[(size_t)q];                             // zr
            res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));
            rtol[(size_t)q] = tol * (normb[(size_t)q] == 0.0 ? 1.0 : normb[(size_t)q]);
            if (res[(size_t)q].back() < rtol[(size_t)q]) stop(q, 0, AMGB_REASON_NONE);
        }
        while (act != 0) {
            RET(M.dot(p, p, 0));
            RET(M.read(1));
            for (int q = 0; q < w; q++) {
                alpha[(size_t)q] = on(q) ? sc[(size_t)q] / M.got[(size_t)q] : 0.0;
                neg_alpha[(size_t)q] = -alpha[(size_t)q];
            }
            RET(M.axpby(alpha.data(), p, ones.data(), xk, act));          // x += alpha p
            if ((it % 8) != 0 && it > 0) {
                RET(many_spmv<K>(h, OP_SPMV, M.A0, p, nullptr, tmp));
                RET(M.axpby(neg_alpha.data(), tmp, ones.data(), r, act)); // r -= alpha A p
            } else {
                RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));          // r = b - A x
            }
            RET(M.precond());                                             // z = M r
            RET(M.dot(z_out, r, 0));
            RET(M.dot(r, r, 1));
            RET(M.read(2));
            for (int q = 0; q < w; q++) {
                if (!on(q)) continue;
                beta[(size_t)q] = M.got[(size_t)q] / sc[(size_t)q];
                sc[(size_t)q] = M.got[(size_t)q];
            }
            RET(many_spmv<K>(h, OP_SPMV, At, z_out, nullptr, tmp));
            RET(M.axpby(ones.data(), tmp, beta.data(), p, act));          // p = beta p + A^H z
            it++;
            for (int q = 0; q < w; q++) {
                if (!on(q)) continue;
                res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));
                if (res[(size_t)q].back() < rtol[(size_t)q]) stop(q, 0, AMGB_REASON_NONE);
                else if (it == maxiter) stop(q, it, AMGB_REASON_NONE);
            }
        }
    } else if (method == AMGB_KRYLOV_MR) {
        double *z = u;
        RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, Vb));                // r = b - A x
        RET(M.precond());                                                 // z = M r
        RET(M.copy(z, z_out));
        RET(M.dot(z, z, 0));
        RET(M.read(1));
        for (int q = 0; q < w; q++) res[(size_t)q].push_back(std::sqrt(M.got[(size_t)q]));
        bool any_b = false;
        for (int q = 0; q < w; q++) any_b = any_b || normb[(size_t)q] != 0.0;
        if (any_b) {                                                      // ||M b||; 1 where b = 0
            RET(M.copy(Vb, bk));
            RET(M.precond());
            RET(M.dot(z_out, z_out, 0));
            RET(M.read(1));
        }
        for (int q = 0; q < w; q++) {
            rtol[(size_t)q] = tol * (normb[(size_t)q] == 0.0 ? 1.0 : std::sqrt(M.got[(size_t)q]));
            if (res[(size_t)q].back() < rtol[(size_t)q]) stop(q, 0, AMGB_REASON_NONE);
        }
        while (act != 0) {
            RET(many_spmv<K>(h, OP_SPMV, M.A0, z, nullptr, Vb));
            RET(M.precond());                                             // p = M (A z)
            RET(M.dot(z_out, z, 0));
            RET(M.dot(z_out, z_out, 1));
            RET(M.read(2));
            for (int q = 0; q < w; q++) {
                if (!on(q)) continue;
                const double pz = M.got[(size_t)q];
                if (pz < 0.0) { stop(q, -1, AMGB_REASON_INDEFINITE_MATRIX); continue; }
                alpha[(size_t)q] = pz / M.got[(size_t)K + q];
                neg_alpha[(size_t)q] = -alpha[(size_t)q];
            }
            if (act == 0) break;
            RET(M.axpby(alpha.data(), z, ones.data(), xk, act));          // x = x + alpha z
            it++;
            if ((it % 50) != 0) {                                         // (sic) recompute on all but every 50th
                RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, Vb));         // r = b - A x
                RET(M.precond());                                         // z = M r
                RET(M.copy(z, z_out));
            } else {
                RET(M.axpby(neg_alpha.data(), z_out, ones.data(), z, act));   // z = z - alpha p
            }
            RET(M.dot(z, z, 0));
            RET(M.read(1));
            for (int q = 0; q < w; q++) {
                if (!on(q)) continue;
                res[(size_t)q].push_back(std::sqrt(M.got[(size_t)q]));
                if (res[(size_t)q].back() < rtol[(size_t)q]) stop(q, 0, AMGB_REASON_NONE);
                else if (it == maxiter) stop(q, it, AMGB_REASON_NONE);
            }
        }
    } else {
        double *r = Vb, *q_ = u;
        RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));                 // r = b - A x
        RET(M.precond());                                                 // z = M r
        RET(M.dot(r, z_out, 0));
        RET(M.dot(r, r, 1));
        RET(M.read(2));
        for (int q = 0; q < w; q++) {
            sc[(size_t)q] = M.got[(size_t)q];                             // rz
            res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));
            rtol[(size_t)q] = tol * (normb[(size_t)q] == 0.0 ? 1.0 : normb[(size_t)q]);
        }
        while (act != 0) {
            RET(many_spmv<K>(h, OP_SPMV, M.A0, z_out, nullptr, q_));     // q = A z
            RET(M.dot(z_out, q_, 0));
            RET(M.read(1));
            for (int q = 0; q < w; q++) {
                if (!on(q)) continue;
                const double zAz = M.got[(size_t)q];
                if (zAz < 0.0) { stop(q, -1, AMGB_REASON_INDEFINITE_MATRIX); continue; }
                alpha[(size_t)q] = sc[(size_t)q] / zAz;
                neg_alpha[(size_t)q] = -alpha[(size_t)q];
            }
            if (act == 0) break;
            RET(M.axpby(alpha.data(), z_out, ones.data(), xk, act));      // x = x + alpha z
            it++;
            if ((it % 50) != 0) RET(many_spmv<K>(h, OP_RESID, M.A0, xk, bk, r));   // (sic) r = b - A x
            else RET(M.axpby(neg_alpha.data(), q_, ones.data(), r, act));           // r = r - alpha q
            RET(M.precond());                                             // z = M r
            RET(M.dot(r, z_out, 0));
            RET(M.dot(r, r, 1));
            RET(M.read(2));
            for (int q = 0; q < w; q++) {
                if (!on(q)) continue;
                sc[(size_t)q] = M.got[(size_t)q];
                if (sc[(size_t)q] < 0.0) { stop(q, -1, AMGB_REASON_INDEFINITE_PRECONDITIONER); continue; }
                res[(size_t)q].push_back(std::sqrt(M.got[(size_t)K + q]));
                if (res[(size_t)q].back() < rtol[(size_t)q]) stop(q, 0, AMGB_REASON_NONE);
                else if (sc[(size_t)q] == 0.0) stop(q, -1, AMGB_REASON_SINGULAR_PRECONDITIONER);
                else if (it == maxiter) stop(q, it, AMGB_REASON_NONE);
            }
        }
    }
    RET(M.store(xk, k, c0, w, X));
    many_krylov_out(k, c0, w, res, status, residuals, n_residuals, info);
    if (reason != nullptr)
        for (int q = 0; q < w; q++) reason[c0 + q] = why[(size_t)q];
    return AMGB_OK;
}

extern "C" int amgb_solve_many_krylov(amgb_hierarchy *h, int32_t method, int32_t k, const double *B_host,
                                      double *X_host, double tol, int32_t maxiter, int32_t cycle, int32_t flags,
                                      double *residuals, int32_t *n_residuals, int32_t *info, int32_t *reason)
{
    RET(check_many_args(h, k, cycle, 1, B_host, X_host));
    if (method < AMGB_KRYLOV_CGNR || method > AMGB_KRYLOV_SD) return fail(AMGB_EINVAL, "unknown Krylov method");
    if (maxiter < 1) return fail(AMGB_EINVAL, "Number of iterations must be positive");
    if ((method == AMGB_KRYLOV_CGNR || method == AMGB_KRYLOV_CGNE) && h->At0.Ap == nullptr)
        return fail(AMGB_ESTATE, "CGNR / CGNE: amgb_hierarchy_set_transpose0 first");
    CallerIo io(h, flags);
    RET(io.begin(B_host, X_host));
    const bool x0_zero = (flags & AMGB_FLAG_X0_ZERO) != 0;
    h->launches = 0;
    for (int c0 = 0; c0 < k; c0 += 8) {
        const int w = std::min(8, k - c0);
        switch (many_width(w)) {
        case 2: RET(many_more_group<2>(method, h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                       residuals, n_residuals, info, reason)); break;
        case 4: RET(many_more_group<4>(method, h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                       residuals, n_residuals, info, reason)); break;
        default: RET(many_more_group<8>(method, h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                        residuals, n_residuals, info, reason)); break;
        }
    }
    h->last_launches = h->launches;
    return io.end();
}
