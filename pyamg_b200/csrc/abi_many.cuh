// abi_many.cuh -- amgb_solve_many / amgb_solve_many_device: MultilevelSolver.solve on up to eight right-hand sides
// per pass over the hierarchy (included by engine.cu).
//
// The operator stream of a cycle (12 B per stored entry of A, P and R) is the same for every right-hand side; a
// batched cycle reads it once for K columns.  Columns run in groups of at most 8; a group of width w is padded to
// K = 2, 4 or 8 with zero columns (a zero right-hand side with a zero iterate stays exactly zero through every
// operation below).  Column j of the result is what amgb_solve_ex computes on that column: every kernel keeps the
// per-row summation order of the single-vector kernel the same operator uses (multi_rhs_kernels.cuh).
//
// Scope: smoothers none / Jacobi / Gauss-Seidel (SOR, any sweep, lexicographic or multi-colour waves) / block Jacobi
// and block Gauss-Seidel (blocksize <= 8) / polynomial (Chebyshev, Richardson) / the normal-equation smoothers
// (jacobi_ne, gauss_seidel_ne, gauss_seidel_nr) / overlapping Schwarz (schwarz, strength_based_schwarz) whose
// K-wide shared memory (2 * largest subdomain * K doubles per warp) fits the single path's 200 KB bound at the
// widest group of the call; the dense coarse operator, the zero coarse solve and a relaxation coarse solver of one
// of those kinds; V / W / F cycles.  Anything else (indexed, CF / FC (block) Jacobi, larger Schwarz subdomains,
// AMLI) returns AMGB_ENOTIMPL before touching the device, and the caller solves column by column.  The batched cycle
// is always the per-launch chain (captured as one CUDA graph per cycle kind and width): the coarse tail, grid and
// resident modes of the single path do not apply to it.

static inline int many_index(int K) { return K == 2 ? 0 : (K == 4 ? 1 : 2); }
static inline int many_width(int w) { return w <= 2 ? 2 : (w <= 4 ? 4 : 8); }

// dynamic shared memory of one many_schwarz_kernel<K> launch: 2 * max_m * K doubles per warp
static size_t many_schwarz_smem(const Smoother &s, int K)
{
    return (size_t)kSchwarzWarps * 2 * (size_t)std::max(s.sz_max_m, 1) * (size_t)K * sizeof(double);
}
constexpr size_t kManySchwarzMaxSmem = 200 * 1024;     // the single path's bound on schwarz_kernel (make_smoother)

static bool many_smoother_supported(const Smoother &s, int K)
{
    switch (s.kind) {
    case AMGB_SM_NONE:
    case AMGB_SM_JACOBI:
    case AMGB_SM_GAUSS_SEIDEL:
    case AMGB_SM_POLYNOMIAL:
    case AMGB_SM_JACOBI_NE:
    case AMGB_SM_GAUSS_SEIDEL_NE:
    case AMGB_SM_GAUSS_SEIDEL_NR: return true;
    case AMGB_SM_SCHWARZ: return many_schwarz_smem(s, K) <= kManySchwarzMaxSmem;
    case AMGB_SM_BLOCK_JACOBI:
    case AMGB_SM_BLOCK_GAUSS_SEIDEL: return s.bs >= 1 && s.bs <= 8;
    }
    return false;
}

// K: the widest group the call runs (a Schwarz level needs K times the single kernel's shared memory)
static int many_supported(const amgb_hierarchy *h, int32_t cycle, int K)
{
    if (cycle == AMGB_CYCLE_AMLI) return fail(AMGB_ENOTIMPL, "solve_many: AMLI cycles run column by column");
    if (h->coarse_relax && !many_smoother_supported(h->coarse_sm, K))
        return fail(AMGB_ENOTIMPL, "solve_many: this coarse relaxation runs column by column");
    for (const Level &L : h->levels) {
        if (!L.has_pr) continue;
        if (!many_smoother_supported(L.pre, K) || !many_smoother_supported(L.post, K))
            return fail(AMGB_ENOTIMPL, "solve_many: this smoother runs column by column");
    }
    return AMGB_OK;
}

// many_schwarz_kernel<K> may take more than 48 KB of dynamic shared memory: opt in before any launch or graph
// capture.  The attribute is per kernel, not per hierarchy, so it is raised to the common bound (which every
// accepted Schwarz level fits) rather than to this hierarchy's need, and never lowered by a smaller one.
template <int K>
static int many_schwarz_optin(const amgb_hierarchy *h)
{
    bool big = h->coarse_relax && h->coarse_sm.kind == AMGB_SM_SCHWARZ && many_schwarz_smem(h->coarse_sm, K) > 48 * 1024;
    for (const Level &L : h->levels) {
        if (!L.has_pr) continue;
        for (const Smoother *s : {&L.pre, &L.post})
            if (s->kind == AMGB_SM_SCHWARZ && many_schwarz_smem(*s, K) > 48 * 1024) big = true;
    }
    if (big) CK(cudaFuncSetAttribute(many_schwarz_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kManySchwarzMaxSmem));
    return AMGB_OK;
}

// rows of a (device or host) array with row pitches: one cudaMemcpy2DAsync (the emulator copies row by row)
static cudaError_t many_copy_2d(void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t height,
                                cudaMemcpyKind kind, cudaStream_t s)
{
#ifdef AMGB_EMU
    for (size_t r = 0; r < height; r++) {
        const cudaError_t e = cudaMemcpyAsync((char *)dst + r * dpitch, (const char *)src + r * spitch, width, kind, s);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
#else
    return cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, kind, s);
#endif
}

// partial sums per column of the level-0 residual launch (rows kernel: one per block; tile kernel: at most 16 per SM)
static long long many_partials_len(const Settings &S, const DevCsr &A0)
{
    return std::max<long long>(csr_grid(A0.n_rows, A0.lanes), (long long)S.num_sms * 16);
}

// K-wide buffers of every level, on the first batched solve of this width (before any graph capture)
template <int K>
static int many_prepare(amgb_hierarchy *h, int n_norms)
{
    ManyWidth &mw = h->many[many_index(K)];
    if (mw.lv.empty()) {
        std::vector<ManyLevel> lv(h->levels.size());
        for (size_t l = 0; l < h->levels.size(); l++) {
            const long long n = (long long)h->levels[l].A.n_rows * K;
            RET(h->dalloc(&lv[l].x_home, n + 2));
            RET(h->dalloc(&lv[l].xalt, n + 2));
            RET(h->dalloc(&lv[l].b, n + 2));
            RET(h->dalloc(&lv[l].r, n + 2));
            lv[l].x = lv[l].x_home;
            if (h->levels[l].poly[0] != nullptr) {   // the level smooths (or coarse-solves) with a polynomial
                RET(h->dalloc(&lv[l].poly[0], n + 2));
                RET(h->dalloc(&lv[l].poly[1], n + 2));
            }
        }
        const DevCsr &A0 = h->levels[0].A;
        RET(h->dalloc(&mw.partials, many_partials_len(h->S, A0) * K));
        RET(h->dalloc(&mw.io, (long long)A0.n_rows * K));
        RET(many_schwarz_optin<K>(h));
        mw.lv = lv;
    }
    if (n_norms > mw.norms2_cap) {
        h->dfree(mw.norms2);
        mw.norms2_cap = std::max(n_norms, 128);
        RET(h->dalloc(&mw.norms2, (long long)mw.norms2_cap * K));
    }
    return AMGB_OK;
}

template <int K, int OP>
static int many_launch(const ManyArgs &a, bool tiles, int grid, cudaStream_t s)
{
    if (tiles) many_tile_kernel<K, OP><<<grid, kManyTileWarps * 32, 0, s>>>(a);
    else many_rows_kernel<K, OP><<<grid, kCsrThreads, 0, s>>>(a);
    CK(cudaGetLastError());
    return AMGB_OK;
}

// *grid_used: blocks launched (= partial sums written), 0 if nothing was launched
template <int K>
static int many_dispatch(const Settings &S, int op, const ManyArgs &a, bool tiles, cudaStream_t s, int *grid_used = nullptr)
{
    long long grid = 0;
    if (tiles) {
        const long long need = (a.tile_end - a.tile_begin + kManyTileWarps - 1) / kManyTileWarps;
        grid = std::min<long long>(need, (long long)S.num_sms * 16);
    } else {
        grid = a.n > 0 ? csr_grid(a.n, a.G) : 0;
        if (grid > 2147483647LL) return fail(AMGB_EINVAL, "launch grid too large");
    }
    if (grid_used) *grid_used = (int)grid;
    if (grid <= 0) return AMGB_OK;
    switch (op) {
    case OP_SPMV: return many_launch<K, OP_SPMV>(a, tiles, (int)grid, s);
    case OP_RESID: return many_launch<K, OP_RESID>(a, tiles, (int)grid, s);
    case OP_PADD: return many_launch<K, OP_PADD>(a, tiles, (int)grid, s);
    case OP_JACOBI: return many_launch<K, OP_JACOBI>(a, tiles, (int)grid, s);
    case OP_GS: return many_launch<K, OP_GS>(a, tiles, (int)grid, s);
    }
    return fail(AMGB_EINVAL, "unknown csr op");
}

static ManyArgs many_args(const Settings &S, const DevCsr &M, const double *x, const double *b, double *y, double omega)
{
    ManyArgs a = {};
    a.Ap = M.Ap; a.Aj = M.Aj; a.Ax = M.Ax;
    a.x = x; a.b = b; a.y = y; a.omega = omega;
    a.T = M.tile_cfg == 7 ? S.dense_T : S.tile_T;
    return a;
}

// one pass over M (amgb_hierarchy::spmv), with the kernel family and lane width `solve` uses for M
template <int K>
static int many_spmv(amgb_hierarchy *h, int op, const DevCsr &M, const double *x, const double *b, double *y,
                     double omega = 0.0, double *parts = nullptr, int *grid_used = nullptr)
{
    if (M.n_rows <= 0) return AMGB_OK;
    h->launches++;
    ManyArgs a = many_args(h->S, M, x, b, y, omega);
    a.partials = parts;
    const bool tiles = M.tiles != nullptr && (M.nnz >= h->S.tile_min_nnz || parts != nullptr);
    if (tiles) {
        a.tiles = M.tiles; a.tile_begin = 0; a.tile_end = M.n_tiles; a.G = M.tile_G;
    } else {
        a.n = M.n_rows; a.row0 = 0; a.rows = nullptr; a.G = M.lanes;
    }
    return many_dispatch<K>(h->S, op, a, tiles, h->stream, grid_used);
}

// one wave of a Gauss-Seidel sweep (amgb_hierarchy::gs_wave)
template <int K>
static int many_gs_wave(amgb_hierarchy *h, const DevCsr &A, const WaveSchedule &ws, long long w, double *x,
                        const double *b, double omega)
{
    const long long p0 = ws.ptr[(size_t)w], nrow = ws.ptr[(size_t)w + 1] - p0;
    if (nrow <= 0) return AMGB_OK;
    h->launches++;
    ManyArgs a = many_args(h->S, A, x, b, x, omega);
    const bool tiles = ws.contiguous && A.tiles != nullptr && ws.nnz[(size_t)w] >= h->S.tile_min_nnz;
    if (tiles) {
        a.tiles = A.tiles; a.tile_begin = ws.tile_ptr[(size_t)w]; a.tile_end = ws.tile_ptr[(size_t)w + 1]; a.G = A.tile_G;
    } else {
        a.n = (int)nrow; a.row0 = ws.contiguous ? (int)p0 : 0; a.rows = ws.contiguous ? nullptr : ws.rows + p0;
        a.G = A.lanes;
    }
    return many_dispatch<K>(h->S, OP_GS, a, tiles, h->stream);
}

template <int K, int BS>
static int many_block_jacobi_bs(int lanes, int nb, const DevCsr &A, const double *x, const double *b,
                                const double *Dinv, double *y, double omega, cudaStream_t s)
{
    if (nb <= 0) return AMGB_OK;
    many_block_jacobi_kernel<K, BS><<<(unsigned)csr_grid(nb, lanes), kCsrThreads, 0, s>>>(lanes, nb, A.Ap, A.Aj, A.Ax, x, b,
                                                                                        Dinv, y, omega);
    CK(cudaGetLastError());
    return AMGB_OK;
}

template <int K>
static int many_block_jacobi(int bs, int lanes, int nb, const DevCsr &A, const double *x, const double *b,
                             const double *Dinv, double *y, double omega, cudaStream_t s)
{
    switch (bs) {
    case 1: return many_block_jacobi_bs<K, 1>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 2: return many_block_jacobi_bs<K, 2>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 3: return many_block_jacobi_bs<K, 3>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 4: return many_block_jacobi_bs<K, 4>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 5: return many_block_jacobi_bs<K, 5>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 6: return many_block_jacobi_bs<K, 6>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 7: return many_block_jacobi_bs<K, 7>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 8: return many_block_jacobi_bs<K, 8>(lanes, nb, A, x, b, Dinv, y, omega, s);
    }
    return fail(AMGB_ENOTIMPL, "block_jacobi: blocksize must be 1..8");
}

template <int K, int BS>
static int many_block_gs_bs(int lanes, int nrows, const int *brows, const DevCsr &A, double *x, const double *b,
                            const double *Dinv, cudaStream_t s)
{
    many_block_gs_kernel<K, BS><<<(unsigned)csr_grid(nrows, lanes), kCsrThreads, 0, s>>>(lanes, nrows, brows, A.Ap, A.Aj,
                                                                                        A.Ax, x, b, Dinv);
    CK(cudaGetLastError());
    return AMGB_OK;
}

// one wave of a block Gauss-Seidel sweep (the `wave` of amgb_hierarchy::block_gauss_seidel)
template <int K>
static int many_block_gs_wave(amgb_hierarchy *h, const DevCsr &A, const Smoother &s, long long w, double *x,
                              const double *b)
{
    const int nrows = (int)(s.ws.ptr[(size_t)w + 1] - s.ws.ptr[(size_t)w]);
    if (nrows <= 0) return AMGB_OK;
    h->launches++;
    const int *brows = s.ws.rows + s.ws.ptr[(size_t)w];
    switch (s.bs) {
    case 1: return many_block_gs_bs<K, 1>(A.lanes, nrows, brows, A, x, b, s.Dinv, h->stream);
    case 2: return many_block_gs_bs<K, 2>(A.lanes, nrows, brows, A, x, b, s.Dinv, h->stream);
    case 3: return many_block_gs_bs<K, 3>(A.lanes, nrows, brows, A, x, b, s.Dinv, h->stream);
    case 4: return many_block_gs_bs<K, 4>(A.lanes, nrows, brows, A, x, b, s.Dinv, h->stream);
    case 5: return many_block_gs_bs<K, 5>(A.lanes, nrows, brows, A, x, b, s.Dinv, h->stream);
    case 6: return many_block_gs_bs<K, 6>(A.lanes, nrows, brows, A, x, b, s.Dinv, h->stream);
    case 7: return many_block_gs_bs<K, 7>(A.lanes, nrows, brows, A, x, b, s.Dinv, h->stream);
    case 8: return many_block_gs_bs<K, 8>(A.lanes, nrows, brows, A, x, b, s.Dinv, h->stream);
    }
    return fail(AMGB_ENOTIMPL, "block_gauss_seidel: blocksize must be 1..8");
}

// amgb_hierarchy::polynomial on the K-wide blocks.  The coefficients are the same for every column and the vector
// passes are elementwise, so they are the single path's scale_kernel / axpby_kernel on the flat n*K array: each
// entry gets the single path's expression, and a zero column stays zero (c*0 + A*0).
template <int K>
static int many_polynomial(amgb_hierarchy *h, Level &L, ManyLevel &V, const Smoother &s)
{
    if (s.coef.empty() || V.poly[0] == nullptr) return fail(AMGB_ESTATE, "polynomial smoother not prepared");
    const long long nk = (long long)L.A.n_rows * K;
    for (int it = 0; it < s.iterations; it++) {
        RET(many_spmv<K>(h, OP_RESID, L.A, V.x, V.b, V.r));
        double *hv = V.poly[0], *Ah = V.poly[1];
        RET(h->scale_to(hv, s.coef[0], V.r, nk));
        for (size_t k = 1; k < s.coef.size(); k++) {
            RET(many_spmv<K>(h, OP_SPMV, L.A, hv, nullptr, Ah));
            RET(h->axpby(s.coef[k], V.r, 1.0, Ah, nk));      // A h + c_k r
            std::swap(hv, Ah);
        }
        RET(h->axpby(1.0, hv, 1.0, V.x, nk));
    }
    return AMGB_OK;
}

template <int K, bool NR>
static int many_kaczmarz(int lanes, int nrows, const int *rows, const DevCsr &M, double *v, const double *b,
                         const double *Dinv, double omega, double *xout, cudaStream_t s)
{
    if (nrows <= 0) return AMGB_OK;
    const dim3 g((unsigned)csr_grid(nrows, lanes)), t(kCsrThreads);
    switch (lanes) {
    case 1: many_kaczmarz_kernel<K, 1, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    case 2: many_kaczmarz_kernel<K, 2, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    case 4: many_kaczmarz_kernel<K, 4, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    case 8: many_kaczmarz_kernel<K, 8, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    case 16: many_kaczmarz_kernel<K, 16, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    default: many_kaczmarz_kernel<K, 32, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    }
    CK(cudaGetLastError());
    return AMGB_OK;
}

// amgb_hierarchy::normal_equations on the K-wide blocks (jacobi_ne / gauss_seidel_ne / gauss_seidel_nr): the same
// launches in the same order, V.r standing for L.r (the NR residual, jacobi_ne's delta)
template <int K>
static int many_normal_equations(amgb_hierarchy *h, Level &L, ManyLevel &V, const Smoother &s)
{
    const long long nk = (long long)L.A.n_rows * K;
    if (s.kind == AMGB_SM_JACOBI_NE) {                                   // relaxation.py:806-812
        double *temp = (V.x == V.x_home) ? V.xalt : V.x_home;
        const unsigned grid = vec_grid(h->S, nk);
        for (int it = 0; it < s.iterations; it++) {
            RET(many_spmv<K>(h, OP_RESID, s.ne_A, V.x, V.b, V.r));       // b - A x
            if (nk > 0) {
                many_mul_rows_kernel<K><<<grid, 256, 0, h->stream>>>(V.r, s.Dinv, nk);             // delta = (b - A x) Dinv
                CK(cudaGetLastError());
            }
            h->launches++;
            RET(many_spmv<K>(h, OP_SPMV, s.ne_At, V.r, nullptr, temp)); // temp = (omega A^H) delta
            RET(h->axpby(1.0, temp, 1.0, V.x, nk));                      // x += temp
        }
        return AMGB_OK;
    }
    const bool nr = s.kind == AMGB_SM_GAUSS_SEIDEL_NR;
    const DevCsr &M = nr ? s.ne_At : s.ne_A;
    const long long nw = (long long)s.ws.ptr.size() - 1;
    auto sweep = [&](bool forward) -> int {
        for (long long q = 0; q < nw; q++) {
            const long long w = forward ? q : nw - 1 - q;
            const int nrow = (int)(s.ws.ptr[(size_t)w + 1] - s.ws.ptr[(size_t)w]);
            const int *rows = s.ws.rows + s.ws.ptr[(size_t)w];
            h->launches++;
            if (nr) RET((many_kaczmarz<K, true>(M.lanes, nrow, rows, M, V.r, nullptr, s.Dinv, s.omega, V.x, h->stream)));
            else RET((many_kaczmarz<K, false>(M.lanes, nrow, rows, M, V.x, V.b, s.Dinv, s.omega, nullptr, h->stream)));
        }
        return AMGB_OK;
    };
    auto residual = [&]() -> int { return nr ? many_spmv<K>(h, OP_RESID, s.ne_A, V.x, V.b, V.r) : AMGB_OK; };
    if (s.sweep == AMGB_SWEEP_SYMMETRIC) {                               // fwd call, then bwd call
        for (int it = 0; it < s.iterations; it++) {
            RET(residual()); RET(sweep(true));
            RET(residual()); RET(sweep(false));
        }
        return AMGB_OK;
    }
    RET(residual());                                                     // once per call, kept up to date by the sweeps
    for (int it = 0; it < s.iterations; it++) RET(sweep(s.sweep == AMGB_SWEEP_FORWARD));
    return AMGB_OK;
}

// amgb_hierarchy::schwarz on the K-wide blocks (many_supported checked the shared memory against the bound, and
// many_prepare opted in above 48 KB)
template <int K>
static int many_schwarz(amgb_hierarchy *h, ManyLevel &V, const Smoother &s)
{
    const long long nw = (long long)s.ws.ptr.size() - 1;
    const size_t smem = many_schwarz_smem(s, K);
    auto sweep = [&](bool forward) -> int {
        for (long long q = 0; q < nw; q++) {
            const long long w = forward ? q : nw - 1 - q;
            const int nd = (int)(s.ws.ptr[(size_t)w + 1] - s.ws.ptr[(size_t)w]);
            if (nd <= 0) continue;
            many_schwarz_kernel<K><<<(unsigned)((nd + kSchwarzWarps - 1) / kSchwarzWarps), kSchwarzWarps * 32, smem,
                                     h->stream>>>(nd, s.ws.rows + s.ws.ptr[(size_t)w], s.sz_Sp, s.sz_Sj, s.sz_Tp, s.Dinv,
                                                  s.ne_A.Ap, s.ne_A.Aj, s.ne_A.Ax, V.x, V.b, std::max(s.sz_max_m, 1));
            CK(cudaGetLastError());
            h->launches++;
        }
        return AMGB_OK;
    };
    for (int it = 0; it < s.iterations; it++) {                          // relaxation.py:241-262
        if (s.sweep == AMGB_SWEEP_FORWARD || s.sweep == AMGB_SWEEP_SYMMETRIC) RET(sweep(true));
        if (s.sweep == AMGB_SWEEP_BACKWARD || s.sweep == AMGB_SWEEP_SYMMETRIC) RET(sweep(false));
    }
    return AMGB_OK;
}

// amgb_hierarchy::smooth for the batched kinds (many_supported rejected the others)
template <int K>
static int many_smooth(amgb_hierarchy *h, Level &L, ManyLevel &V, const Smoother &s)
{
    switch (s.kind) {
    case AMGB_SM_NONE: return AMGB_OK;
    case AMGB_SM_JACOBI:
        for (int it = 0; it < s.iterations; it++) {
            RET(many_spmv<K>(h, OP_JACOBI, L.A, V.x, V.b, V.xalt, s.omega));
            std::swap(V.x, V.xalt);
        }
        return AMGB_OK;
    case AMGB_SM_GAUSS_SEIDEL: {
        const long long nw = (long long)s.ws.ptr.size() - 1;
        const double om = (s.sweep == AMGB_SWEEP_SYMMETRIC) ? 1.0 : s.omega;   // relaxation.py:326-330
        for (int it = 0; it < s.iterations; it++) {
            if (s.sweep == AMGB_SWEEP_FORWARD || s.sweep == AMGB_SWEEP_SYMMETRIC)
                for (long long w = 0; w < nw; w++) RET(many_gs_wave<K>(h, L.A, s.ws, w, V.x, V.b, om));
            if (s.sweep == AMGB_SWEEP_BACKWARD)
                for (long long w = nw - 1; w >= 0; w--) RET(many_gs_wave<K>(h, L.A, s.ws, w, V.x, V.b, om));
            if (s.sweep == AMGB_SWEEP_SYMMETRIC)      // the idempotent middle wave is skipped, as in smooth()
                for (long long w = nw - 2; w >= 0; w--) RET(many_gs_wave<K>(h, L.A, s.ws, w, V.x, V.b, om));
        }
        return AMGB_OK;
    }
    case AMGB_SM_BLOCK_JACOBI:
        for (int it = 0; it < s.iterations; it++) {
            h->launches++;
            RET(many_block_jacobi<K>(s.bs, L.A.lanes, L.A.n_rows / s.bs, L.A, V.x, V.b, s.Dinv, V.xalt, s.omega,
                                     h->stream));
            std::swap(V.x, V.xalt);
        }
        return AMGB_OK;
    case AMGB_SM_BLOCK_GAUSS_SEIDEL: {
        const long long nw = (long long)s.ws.ptr.size() - 1;
        for (int it = 0; it < s.iterations; it++) {
            if (s.sweep == AMGB_SWEEP_FORWARD || s.sweep == AMGB_SWEEP_SYMMETRIC)
                for (long long w = 0; w < nw; w++) RET(many_block_gs_wave<K>(h, L.A, s, w, V.x, V.b));
            if (s.sweep == AMGB_SWEEP_BACKWARD)
                for (long long w = nw - 1; w >= 0; w--) RET(many_block_gs_wave<K>(h, L.A, s, w, V.x, V.b));
            if (s.sweep == AMGB_SWEEP_SYMMETRIC)      // the idempotent middle wave is skipped, as in block_gauss_seidel()
                for (long long w = nw - 2; w >= 0; w--) RET(many_block_gs_wave<K>(h, L.A, s, w, V.x, V.b));
        }
        return AMGB_OK;
    }
    case AMGB_SM_POLYNOMIAL: return many_polynomial<K>(h, L, V, s);
    case AMGB_SM_JACOBI_NE:
    case AMGB_SM_GAUSS_SEIDEL_NE:
    case AMGB_SM_GAUSS_SEIDEL_NR: return many_normal_equations<K>(h, L, V, s);
    case AMGB_SM_SCHWARZ: return many_schwarz<K>(h, V, s);
    }
    return fail(AMGB_ENOTIMPL, "solve_many: smoother kind");
}

// multilevel.py:617-618 / :559-561 (amgb_hierarchy::coarse_solve): zero when the coarsest A has no entries, a
// relaxation from zero, or the dense coarse operator
template <int K>
static int many_coarse(amgb_hierarchy *h, Level &Lc, ManyLevel &V)
{
    if (h->coarse_zero) return h->launch_count_fill(V.x, (long long)Lc.A.n_rows * K);
    if (h->coarse_relax) {                                              // :773-779
        const long long nk = (long long)Lc.A.n_rows * K;
        V.x = V.x_home;
        RET(h->launch_count_fill(V.x, nk));
        RET(many_smooth<K>(h, Lc, V, h->coarse_sm));
        if (V.x != V.x_home) {                                          // odd number of Jacobi ping-pongs
            CK(cudaMemcpyAsync(V.x_home, V.x, sizeof(double) * (size_t)nk, cudaMemcpyDeviceToDevice, h->stream));
            h->launches++;
            std::swap(V.x, V.xalt);
        }
        return AMGB_OK;
    }
    const int n = h->coarse_n, threads = 128, rows_per_block = threads / 32;
    many_dense_matvec_kernel<K><<<(n + rows_per_block - 1) / rows_per_block, threads, 0, h->stream>>>(n, n, h->coarse_pinv,
                                                                                                   V.b, V.x);
    CK(cudaGetLastError());
    h->launches++;
    return AMGB_OK;
}

template <int K>
static int many_cycle(amgb_hierarchy *h, std::vector<ManyLevel> &lv, int lvl, int kind, int cpl);

// multilevel.py:615-629
template <int K>
static int many_descend(amgb_hierarchy *h, std::vector<ManyLevel> &lv, int lvl, int kind, int cpl)
{
    Level &C = h->levels[(size_t)lvl + 1];
    ManyLevel &W = lv[(size_t)lvl + 1];
    if (lvl == (int)h->levels.size() - 2) return many_coarse<K>(h, C, W);
    RET(h->launch_count_fill(W.x, (long long)C.A.n_rows * K));
    if (kind == AMGB_CYCLE_V) {
        RET(many_cycle<K>(h, lv, lvl + 1, AMGB_CYCLE_V, 1));
    } else if (kind == AMGB_CYCLE_W) {
        RET(many_cycle<K>(h, lv, lvl + 1, kind, cpl));
        RET(many_cycle<K>(h, lv, lvl + 1, kind, cpl));
    } else {
        RET(many_cycle<K>(h, lv, lvl + 1, kind, cpl));
        for (int q = 0; q < cpl; q++) RET(many_cycle<K>(h, lv, lvl + 1, AMGB_CYCLE_V, 1));
    }
    return AMGB_OK;
}

// multilevel.py:584-662 on K columns (amgb_hierarchy::cycle)
template <int K>
static int many_cycle(amgb_hierarchy *h, std::vector<ManyLevel> &lv, int lvl, int kind, int cpl)
{
    Level &L = h->levels[(size_t)lvl];
    ManyLevel &V = lv[(size_t)lvl];
    ManyLevel &W = lv[(size_t)lvl + 1];
    RET(many_smooth<K>(h, L, V, L.pre));
    RET(many_spmv<K>(h, OP_RESID, L.A, V.x, V.b, V.r));
    RET(many_spmv<K>(h, OP_SPMV, L.R, V.r, nullptr, W.b));
    RET(many_descend<K>(h, lv, lvl, kind, cpl));
    RET(many_spmv<K>(h, OP_PADD, L.P, W.x, nullptr, V.x));
    RET(many_smooth<K>(h, L, V, L.post));
    if (V.x != V.x_home) {   // odd number of Jacobi ping-pongs: bring the iterate home
        CK(cudaMemcpyAsync(V.x_home, V.x, sizeof(double) * (size_t)L.A.n_rows * K, cudaMemcpyDeviceToDevice, h->stream));
        h->launches++;
        std::swap(V.x, V.xalt);
    }
    return AMGB_OK;
}

// amgb_hierarchy::one_iteration: one CUDA graph per (cycle kind, K)
template <int K>
static int many_one_iteration(amgb_hierarchy *h, int kind, int cpl)
{
    ManyWidth &mw = h->many[many_index(K)];
    if (h->levels.size() == 1) return many_coarse<K>(h, h->levels[0], mw.lv[0]);
    if (!h->S.use_graph) return many_cycle<K>(h, mw.lv, 0, kind, cpl);
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(h->stream, &st) == cudaSuccess && st == cudaStreamCaptureStatusActive)
        return many_cycle<K>(h, mw.lv, 0, kind, cpl);
    if (mw.graph[kind] == nullptr || mw.graph_cpl[kind] != cpl) {
        if (mw.graph[kind] != nullptr) { cudaGraphExecDestroy(mw.graph[kind]); mw.graph[kind] = nullptr; }
        const long long before = h->launches;
        cudaGraph_t g = nullptr;
        CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
        const int rc = many_cycle<K>(h, mw.lv, 0, kind, cpl);
        const cudaError_t e = cudaStreamEndCapture(h->stream, &g);
        if (rc != AMGB_OK) { if (g) cudaGraphDestroy(g); return rc; }
        if (e != cudaSuccess) return fail(AMGB_ECUDA, std::string("graph capture: ") + cudaGetErrorString(e));
        mw.graph_nodes[kind] = h->launches - before;
        h->launches = before;
        CK(cudaGraphInstantiate(&mw.graph[kind], g, 0));
        cudaGraphDestroy(g);
        mw.graph_cpl[kind] = cpl;
    }
    CK(cudaGraphLaunch(mw.graph[kind], h->stream));
    h->launches += mw.graph_nodes[kind];
    return AMGB_OK;
}

// ||b - A x||^2 of the K level-0 columns -> norms2[slot*K .. slot*K+K)
template <int K>
static int many_residual_norm2(amgb_hierarchy *h, int slot)
{
    ManyWidth &mw = h->many[many_index(K)];
    ManyLevel &V = mw.lv[0];
    int grid = 0;
    RET(many_spmv<K>(h, OP_RESID, h->levels[0].A, V.x, V.b, V.r, 0.0, mw.partials, &grid));
    many_reduce_kernel<K><<<1, 1024, 0, h->stream>>>(mw.partials, grid, mw.norms2 + (size_t)slot * K);
    CK(cudaGetLastError());
    h->launches++;
    return AMGB_OK;
}

// ||b||^2 of the K level-0 columns -> norms2[slot*K ..)
template <int K>
static int many_rhs_norm2(amgb_hierarchy *h, int slot)
{
    ManyWidth &mw = h->many[many_index(K)];
    many_sumsq_kernel<K><<<sumsq_blocks(h->S), 256, 0, h->stream>>>(mw.lv[0].b, h->levels[0].A.n_rows, mw.partials);
    CK(cudaGetLastError());
    many_reduce_kernel<K><<<1, 1024, 0, h->stream>>>(mw.partials, sumsq_blocks(h->S), mw.norms2 + (size_t)slot * K);
    CK(cudaGetLastError());
    h->launches += 2;
    return AMGB_OK;
}

// columns [0, w) of the device array src (row pitch ld, caller's row order) -> level-0 block dst, zero-padded
template <int K>
static int many_load(amgb_hierarchy *h, const double *src, long long ld, int w, double *dst)
{
    const long long n = h->levels[0].A.n_rows;
    many_pack_kernel<K><<<vec_grid(h->S, n * K), 256, 0, h->stream>>>(src, ld, w, h->order0, dst, n);
    CK(cudaGetLastError());
    h->launches++;
    return AMGB_OK;
}

// columns [q0, q1) of the level-0 block src -> device array dst (row pitch ld, caller's row order)
template <int K>
static int many_store(amgb_hierarchy *h, const double *src, int q0, int q1, double *dst, long long ld)
{
    const long long n = h->levels[0].A.n_rows;
    if (q1 <= q0) return AMGB_OK;
    many_unpack_kernel<K><<<vec_grid(h->S, n * (q1 - q0)), 256, 0, h->stream>>>(src, h->order0, dst, ld, q0, q1, n);
    CK(cudaGetLastError());
    h->launches++;
    return AMGB_OK;
}

// columns [c0, c0+w) of the caller's n x k arrays through one K-wide group (amgb_solve_ex per column).  Host arrays
// are staged through mw.io; device arrays (dev) are packed from and unpacked into in place.
template <int K>
static int many_group_host(amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X, bool x0_zero,
                           bool dev, double tol, int32_t maxiter, int32_t cycle, int32_t cpl, double *residuals,
                           int32_t *n_residuals, int32_t *info)
{
    RET(many_prepare<K>(h, maxiter + 1));
    ManyWidth &mw = h->many[many_index(K)];
    ManyLevel &V = mw.lv[0];
    const long long n = h->levels[0].A.n_rows;
    cudaStream_t s = h->stream;
    const size_t pitch = sizeof(double) * (size_t)k, wb = sizeof(double) * (size_t)w;
    auto load = [&](const double *src, double *dst) -> int {
        if (dev) return many_load<K>(h, src + c0, k, w, dst);
        CK(many_copy_2d(mw.io, wb, src + c0, pitch, wb, (size_t)n, cudaMemcpyHostToDevice, s));
        return many_load<K>(h, mw.io, w, w, dst);
    };
    double *const out = dev ? X + c0 : mw.io;     // where many_store writes the group's columns, row pitch out_ld
    const long long out_ld = dev ? k : w;
    V.x = V.x_home;
    RET(load(B, V.b));
    if (x0_zero) RET(h->launch_count_fill(V.x, n * K));
    else RET(load(X, V.x));
    std::vector<double> normb((size_t)K, 1.0), got((size_t)K);
    auto read_norms = [&](int slot) -> int {
        CK(cudaMemcpyAsync(got.data(), mw.norms2 + (size_t)slot * K, sizeof(double) * K, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return AMGB_OK;
    };
    // normb (multilevel.py:540-542) per column; with x0 = 0 the initial residual is b itself (:545)
    if (tol > 0.0 || x0_zero) RET(many_rhs_norm2<K>(h, 0));
    if (tol > 0.0) {
        RET(read_norms(0));
        for (int q = 0; q < K; q++) {
            normb[(size_t)q] = std::sqrt(got[(size_t)q]);
            if (normb[(size_t)q] == 0.0) normb[(size_t)q] = 1.0;
        }
    }
    if (!x0_zero) RET(many_residual_norm2<K>(h, 0));
    std::vector<int> conv_at((size_t)w, 0);     // cycle after which column q met the tolerance (0: not yet)
    int it = 0, running = w;
    while (true) {
        RET(many_one_iteration<K>(h, cycle, cpl));                        // :559-563
        it++;
        RET(many_residual_norm2<K>(h, it));                               // :567
        if (tol > 0.0) {
            RET(read_norms(it));
            for (int q = 0; q < w; q++) {
                if (conv_at[(size_t)q] == 0 && std::sqrt(got[(size_t)q]) < tol * normb[(size_t)q]) {   // :574
                    conv_at[(size_t)q] = it;
                    running--;
                    RET(many_store<K>(h, V.x, q, q + 1, out, out_ld));    // this column keeps this iterate
                }
            }
            if (running == 0) break;
        }
        if (it == maxiter) break;                                         // :579
    }
    for (int q = 0; q < w;) {                                             // the columns still running: last iterate
        if (conv_at[(size_t)q] != 0) { q++; continue; }
        int e = q;
        while (e < w && conv_at[(size_t)e] == 0) e++;
        RET(many_store<K>(h, V.x, q, e, out, out_ld));
        q = e;
    }
    std::vector<double> n2;
    if (!dev) CK(many_copy_2d(X + c0, pitch, mw.io, wb, wb, (size_t)n, cudaMemcpyDeviceToHost, s));
    if (!dev || residuals != nullptr) {          // device I/O without a residual list: nothing to wait for
        n2.resize(((size_t)it + 1) * K);
        CK(cudaMemcpyAsync(n2.data(), mw.norms2, sizeof(double) * n2.size(), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    for (int q = 0; q < w; q++) {
        const int last = conv_at[(size_t)q] ? conv_at[(size_t)q] : it;
        if (residuals != nullptr)
            for (int t = 0; t <= last; t++) residuals[(size_t)t * k + c0 + q] = std::sqrt(n2[(size_t)t * K + q]);
        if (n_residuals != nullptr) n_residuals[c0 + q] = last + 1;
        if (info != nullptr) info[c0 + q] = conv_at[(size_t)q] ? 0 : it;
    }
    return AMGB_OK;
}

template <int K>
static int many_group_device(amgb_hierarchy *h, int32_t k, int c0, int w, const double *B, double *X, int32_t ncycles,
                             int32_t cycle, int32_t cpl, double *norms2_dev)
{
    RET(many_prepare<K>(h, ncycles + 1));
    ManyWidth &mw = h->many[many_index(K)];
    ManyLevel &V = mw.lv[0];
    V.x = V.x_home;
    RET(many_load<K>(h, B + c0, k, w, V.b));
    RET(many_load<K>(h, X + c0, k, w, V.x));
    if (norms2_dev != nullptr) RET(many_residual_norm2<K>(h, 0));
    for (int it = 1; it <= ncycles; it++) {
        RET(many_one_iteration<K>(h, cycle, cpl));
        if (norms2_dev != nullptr) RET(many_residual_norm2<K>(h, it));
    }
    RET(many_store<K>(h, V.x, 0, w, X + c0, k));
    if (norms2_dev != nullptr)
        CK(many_copy_2d(norms2_dev + c0, sizeof(double) * (size_t)k, mw.norms2, sizeof(double) * K, sizeof(double) * (size_t)w,
                        (size_t)ncycles + 1, cudaMemcpyDeviceToDevice, h->stream));
    return AMGB_OK;
}

static int check_many_args(amgb_hierarchy *h, int32_t k, int32_t cycle, int32_t cpl, const void *B, const void *X)
{
    RET(check_cycle_args(h, cycle, cpl));
    if (k < 1) return fail(AMGB_EINVAL, "solve_many: k must be >= 1");
    if (B == nullptr || X == nullptr) return fail(AMGB_EINVAL, "null block");
    RET(many_supported(h, cycle, many_width(std::min(k, 8))));
    CK(cudaSetDevice(h->device));
    return AMGB_OK;
}

extern "C" int amgb_solve_many(amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host, double tol,
                               int32_t maxiter, int32_t cycle, int32_t cycles_per_level, int32_t flags,
                               double *residuals, int32_t *n_residuals, int32_t *info)
{
    RET(check_many_args(h, k, cycle, cycles_per_level, B_host, X_host));
    if (maxiter < 1) return fail(AMGB_EINVAL, "maxiter must be >= 1");
    CallerIo io(h, flags);
    RET(io.begin(B_host, X_host));
    const bool x0_zero = (flags & AMGB_FLAG_X0_ZERO) != 0;
    h->launches = 0;
    for (int c0 = 0; c0 < k; c0 += 8) {
        const int w = std::min(8, k - c0);
        switch (many_width(w)) {
        case 2: RET(many_group_host<2>(h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                       cycles_per_level, residuals, n_residuals, info)); break;
        case 4: RET(many_group_host<4>(h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                       cycles_per_level, residuals, n_residuals, info)); break;
        default: RET(many_group_host<8>(h, k, c0, w, B_host, X_host, x0_zero, io.dev, tol, maxiter, cycle,
                                        cycles_per_level, residuals, n_residuals, info)); break;
        }
    }
    h->last_launches = h->launches;
    return io.end();
}

extern "C" int amgb_solve_many_device(amgb_hierarchy *h, int32_t k, const double *B_dev, double *X_dev, int32_t ncycles,
                                      int32_t cycle, int32_t cycles_per_level, double *norms2_dev)
{
    RET(check_many_args(h, k, cycle, cycles_per_level, B_dev, X_dev));
    if (ncycles < 0) return fail(AMGB_EINVAL, "ncycles < 0");
    h->launches = 0;
    for (int c0 = 0; c0 < k; c0 += 8) {
        const int w = std::min(8, k - c0);
        switch (many_width(w)) {
        case 2: RET(many_group_device<2>(h, k, c0, w, B_dev, X_dev, ncycles, cycle, cycles_per_level, norms2_dev)); break;
        case 4: RET(many_group_device<4>(h, k, c0, w, B_dev, X_dev, ncycles, cycle, cycles_per_level, norms2_dev)); break;
        default: RET(many_group_device<8>(h, k, c0, w, B_dev, X_dev, ncycles, cycle, cycles_per_level, norms2_dev)); break;
        }
    }
    h->last_launches = h->launches;
    return AMGB_OK;
}
