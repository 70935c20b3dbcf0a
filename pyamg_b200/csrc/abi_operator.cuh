// abi_operator.cuh -- part of engine.cu's translation unit (included there): resident single operators
// (amgb_operator_*), resident-basis Arnoldi (amgb_arnoldi_*), host-only debug helpers and the device-pointer kernel
// entry points (amgb_dev_*).  Not a stand-alone header.
#pragma once

// ------------------------------------------------------------------------------------------
// C ABI (1b): one resident operator with the tile kernels -- the building block of the multi-GPU layer
// (pyamg_b200/dist.py) and of Krylov-style callers that keep their vectors on the device.
// ------------------------------------------------------------------------------------------
struct amgb_operator {
    amgb_hierarchy *pool = nullptr;      // owns the device allocations
    DevCsr M;
    WaveSchedule waves;                  // optional contiguous wave ranges (Gauss-Seidel)
    double *partials = nullptr;
};

extern "C" int amgb_operator_create(int device, const amgb_matrix *Min, const int64_t *wave_ptr, int32_t n_waves,
                                    void *stream, amgb_operator **out)
{
    if (out == nullptr) return fail(AMGB_EINVAL, "out is null");
    *out = nullptr;
    amgb_hierarchy *pool = nullptr;
    RET(amgb_hierarchy_create(device, &pool));
    std::unique_ptr<amgb_operator> op(new amgb_operator());
    op->pool = pool;
    auto bail = [&](int rc) { amgb_hierarchy_destroy(pool); return rc; };
    HostCsr H;
    int rc = to_host_csr(Min, H, "M");
    if (rc != AMGB_OK) return bail(rc);
    if (stream != nullptr) pool->stream = (cudaStream_t)stream;
    else {
        if (cudaStreamCreateWithFlags(&pool->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(fail(AMGB_ECUDA, "stream"));
        pool->own_stream = true;
    }
    if (wave_ptr != nullptr && n_waves > 0) {
        WaveSchedule &W = op->waves;
        W.ptr.assign(wave_ptr, wave_ptr + n_waves + 1);
        if (W.ptr.front() != 0 || W.ptr.back() > H.n_rows) return bail(fail(AMGB_EINVAL, "wave_ptr out of range"));
        for (int w = 0; w < n_waves; w++)
            if (W.ptr[(size_t)w + 1] < W.ptr[(size_t)w]) return bail(fail(AMGB_EINVAL, "wave_ptr not monotone"));
        W.contiguous = true;
        W.nnz.assign((size_t)n_waves, 0);
        for (int w = 0; w < n_waves; w++)
            W.nnz[(size_t)w] = H.Ap[(size_t)W.ptr[(size_t)w + 1]] - H.Ap[(size_t)W.ptr[(size_t)w]];
        std::vector<long long> breaks(W.ptr);
        if (breaks.back() != H.n_rows) breaks.push_back(H.n_rows);
        rc = pool->upload_csr(H, op->M, &breaks, &W.tile_ptr);
        if (!pool->S.use_tiles) W.tile_ptr.clear();
    } else {
        rc = pool->upload_csr(H, op->M);
    }
    if (rc != AMGB_OK) return bail(rc);
    rc = pool->dalloc(&op->partials, std::max<long long>(pool->partials_len(op->M), 1));
    if (rc != AMGB_OK) return bail(rc);
    *out = op.release();
    return AMGB_OK;
}

extern "C" void amgb_operator_destroy(amgb_operator *op)
{
    if (op == nullptr) return;
    amgb_hierarchy_destroy(op->pool);
    delete op;
}

// kind: 0 y = M x | 1 y = b - M x (norm2_out, if given, receives |y|^2) | 2 y += M x |
//       3 y = jacobi(x; b, omega), r (optional) = b - M x | 4 Gauss-Seidel on wave `wave` of y (= x) in place.
// All pointers are DEVICE pointers; x must have M.n_cols entries (+2 readable doubles of padding).
extern "C" int amgb_operator_apply(amgb_operator *op, int32_t kind, const double *x, const double *b, double *y,
                                   double *r, double omega, double *norm2_out, int32_t wave)
{
    if (op == nullptr) return fail(AMGB_EINVAL, "null operator");
    amgb_hierarchy *h = op->pool;
    CK(cudaSetDevice(h->device));
    if (kind < 0 || kind > 4) return fail(AMGB_EINVAL, "unknown operator kind");
    if (kind == OP_GS) {
        if (wave < 0 || (size_t)wave + 1 >= op->waves.ptr.size()) return fail(AMGB_EINVAL, "wave index out of range");
        return h->gs_wave(op->M, op->waves, wave, y, b, omega);
    }
    double *parts = (norm2_out != nullptr && (kind == OP_RESID || kind == OP_JACOBI)) ? op->partials : nullptr;
    RET(h->spmv(kind, op->M, x, b, y, omega, r, parts));
    if (parts != nullptr) {
        reduce_partials_kernel<<<1, 1024, 0, h->stream>>>(parts, (int)h->partials_used(op->M, kind), norm2_out);
        CK(cudaGetLastError());
    }
    return AMGB_OK;
}

// ------------------------------------------------------------------------------------------
// C ABI (1c): GPU-resident Arnoldi rounds for the spectral-radius estimates of the smoother setup
// (SURVEY.md 8(f)-4; pyamg/util/linalg.py:255-383 approximate_spectral_radius -> _approximate_eigenvalues :90-252:
// rho(D^-1 A) for Jacobi's omega, smoothing.py:372-400, rho(A) for Richardson / Chebyshev, :611-647).
// The operator x -> diag(row_scale) (A x) is uploaded once; one call runs a whole round of modified-Gram-Schmidt
// Arnoldi without a host round trip (inner products stay in device scalars: dot_to + axpy_ratio_kernel), the small
// Hessenberg matrix goes to the host, whose eigen-decomposition (LAPACK through SciPy, as in the reference)
// picks the restart vector as a combination of the basis that is still resident.
// ------------------------------------------------------------------------------------------
struct amgb_arnoldi {
    amgb_hierarchy *pool = nullptr;
    DevCsr M;
    int maxiter = 0;
    long long n = 0, npad = 0;
    double *V = nullptr, *w = nullptr, *scale = nullptr, *dH = nullptr, *one = nullptr;
    bool have_start = false;
    double *v(int j) const { return V + (size_t)j * npad; }
};

extern "C" int amgb_arnoldi_create(int device, const amgb_matrix *A, const double *row_scale, int32_t maxiter,
                                   amgb_arnoldi **out)
{
    if (out == nullptr) return fail(AMGB_EINVAL, "out is null");
    *out = nullptr;
    if (maxiter < 1) return fail(AMGB_EINVAL, "maxiter < 1");
    amgb_hierarchy *pool = nullptr;
    RET(amgb_hierarchy_create(device, &pool));
    std::unique_ptr<amgb_arnoldi> a(new amgb_arnoldi());
    a->pool = pool;
    auto bail = [&](int rc) { amgb_hierarchy_destroy(pool); return rc; };
    HostCsr H;
    int rc = to_host_csr(A, H, "A");
    if (rc == AMGB_OK && H.n_rows != H.n_cols) rc = fail(AMGB_EINVAL, "expected square matrix");   // linalg.py:150-151
    if (rc != AMGB_OK) return bail(rc);
    if (cudaStreamCreateWithFlags(&pool->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(fail(AMGB_ECUDA, "stream"));
    pool->own_stream = true;
    a->n = H.n_rows;
    a->npad = ((a->n + 2 + 31) / 32) * 32;
    a->maxiter = (int)std::min<long long>(maxiter, std::max<long long>(a->n, 1));
    rc = pool->upload_csr(H, a->M);
    if (rc == AMGB_OK) rc = pool->dalloc(&a->V, (long long)(a->maxiter + 1) * a->npad);
    if (rc == AMGB_OK) rc = pool->dalloc(&a->w, a->npad);
    if (rc == AMGB_OK) rc = pool->dalloc(&a->dH, (long long)(a->maxiter + 1) * a->maxiter);
    if (rc == AMGB_OK) rc = pool->dalloc(&a->one, 8);
    if (rc == AMGB_OK) rc = pool->dalloc(&pool->sumsq_parts, kSumsqBlocks);
    if (rc == AMGB_OK && row_scale != nullptr) rc = pool->upload(&a->scale, row_scale, a->n, 2);
    if (rc != AMGB_OK) return bail(rc);
    const double init[2] = {1.0, 0.0};
    if (cudaMemcpy(a->one, init, sizeof init, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemset(a->V, 0, sizeof(double) * (size_t)(a->maxiter + 1) * (size_t)a->npad) != cudaSuccess ||
        cudaMemset(a->w, 0, sizeof(double) * (size_t)a->npad) != cudaSuccess ||
        cudaHostAlloc((void **)&pool->norm_host, sizeof(double) * 2, cudaHostAllocDefault) != cudaSuccess)
        return bail(fail(AMGB_ECUDA, "arnoldi: device initialisation"));
    *out = a.release();
    return AMGB_OK;
}

extern "C" void amgb_arnoldi_destroy(amgb_arnoldi *a)
{
    if (a == nullptr) return;
    amgb_hierarchy_destroy(a->pool);
    delete a;
}

// One round: V[0] = v0 / ||v0|| (v0 from the host, or -- v0_host == NULL -- the vector left by amgb_arnoldi_combine),
// then maxiter steps  w = diag(s) A V[j];  H[i][j] = <V[i], w>, w -= H[i][j] V[i] (i <= j);  H[j+1][j] = ||w||;
// V[j+1] = w / H[j+1][j].  H: (maxiter+1) x maxiter row-major on the host.  *m_done = number of valid steps: the
// first j with H[j+1][j] < breakdown * max(1, max |H[:j+1,:j+1]|) ends the round at m = j + 1 (later columns are
// then meaningless); 0 if the start vector is zero.
extern "C" int amgb_arnoldi_run(amgb_arnoldi *a, const double *v0_host, double breakdown, double *H_host, int32_t *m_done)
{
    if (a == nullptr || H_host == nullptr || m_done == nullptr) return fail(AMGB_EINVAL, "null argument");
    amgb_hierarchy *h = a->pool;
    CK(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    const long long n = a->n;
    const int mi = a->maxiter;
    *m_done = 0;
    if (v0_host != nullptr) CK(cudaMemcpyAsync(a->v(0), v0_host, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, s));
    else if (!a->have_start) return fail(AMGB_ESTATE, "arnoldi: no start vector (call amgb_arnoldi_combine or pass v0)");
    a->have_start = false;
    double *scal = a->one + 1;
    RET(h->dot_to(a->v(0), a->v(0), n, scal));
    CK(cudaMemcpyAsync(h->norm_host, scal, sizeof(double), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (!(h->norm_host[0] > 0.0)) {
        std::fill(H_host, H_host + (size_t)(mi + 1) * mi, 0.0);
        return AMGB_OK;
    }
    const unsigned grid = vec_grid(h->S, n);
    div_kernel<<<grid, 256, 0, s>>>(a->v(0), std::sqrt(h->norm_host[0]), n);
    CK(cudaGetLastError());
    CK(cudaMemsetAsync(a->dH, 0, sizeof(double) * (size_t)(mi + 1) * (size_t)mi, s));
    for (int j = 0; j < mi; j++) {
        RET(h->spmv(OP_SPMV, a->M, a->v(j), nullptr, a->w));
        if (a->scale != nullptr) {
            mul_kernel<<<grid, 256, 0, s>>>(a->w, a->scale, n);
            CK(cudaGetLastError());
        }
        for (int i = 0; i <= j; i++) {
            double *hij = a->dH + (size_t)i * mi + j;
            RET(h->dot_to(a->v(i), a->w, n, hij));
            RET(h->axpy_ratio(a->w, a->v(i), hij, a->one, -1.0, n));
        }
        double *hn = a->dH + (size_t)(j + 1) * mi + j;
        RET(h->dot_to(a->w, a->w, n, hn));
        sqrt_scalar_kernel<<<1, 1, 0, s>>>(hn);
        CK(cudaGetLastError());
        div_dev_kernel<<<grid, 256, 0, s>>>(a->v(j + 1), a->w, hn, n);
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(H_host, a->dH, sizeof(double) * (size_t)(mi + 1) * (size_t)mi, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    int m = mi;
    double hmax = 0.0;
    for (int j = 0; j < mi; j++) {
        for (int i = 0; i <= j; i++) hmax = std::max(hmax, std::fabs(H_host[(size_t)i * mi + j]));
        for (int jj = 0; jj < j; jj++) hmax = std::max(hmax, std::fabs(H_host[(size_t)j * mi + jj]));
        if (!(H_host[(size_t)(j + 1) * mi + j] >= breakdown * std::max(1.0, hmax))) { m = j + 1; break; }
    }
    *m_done = m;
    return AMGB_OK;
}

// next start vector = sum_k coef[k] V[k], k < m (the dominant Ritz vector: linalg.py:369-371)
extern "C" int amgb_arnoldi_combine(amgb_arnoldi *a, const double *coef, int32_t m)
{
    if (a == nullptr || coef == nullptr) return fail(AMGB_EINVAL, "null argument");
    if (m < 1 || m > a->maxiter) return fail(AMGB_EINVAL, "arnoldi: m out of range");
    amgb_hierarchy *h = a->pool;
    CK(cudaSetDevice(h->device));
    RET(h->scale_to(a->w, coef[0], a->v(0), a->n));
    for (int k = 1; k < m; k++) RET(h->axpby(coef[k], a->v(k), 1.0, a->w, a->n));
    RET(h->copy_vec(a->v(0), a->w, a->n));
    a->have_start = true;
    return AMGB_OK;
}

// HOST helper (no CUDA): the tile list the engine would build for a CSR row-pointer array under the
// geometry (T entries, RMAX rows per tile) with G lanes per row and optional row breaks (e.g. wave
// boundaries, n_breaks+1 ascending entries starting at 0).  row0/nz0 receive n_tiles+1 descriptors (sentinel
// last, capacity `cap`), tile_ptr (if non-null, n_breaks+1 entries) the tile range of every break range.
// Exposed so the tiling invariants can be tested without a GPU.
extern "C" int amgb_debug_build_tiles(int32_t n, const int32_t *Ap, int32_t G, const int64_t *breaks,
                                      int32_t n_breaks, int32_t T, int32_t RMAX, int32_t *row0, int32_t *nz0,
                                      int32_t cap, int32_t *tile_ptr, int32_t *n_tiles)
{
    if (Ap == nullptr || row0 == nullptr || nz0 == nullptr || n_tiles == nullptr || n < 0)
        return fail(AMGB_EINVAL, "build_tiles: bad arguments");
    if (G < 1 || G > 32 || (G & (G - 1)) || T < 1 || RMAX < 1) return fail(AMGB_EINVAL, "build_tiles: bad geometry");
    HostCsr H;
    H.n_rows = H.n_cols = n;
    H.Ap.assign(Ap, Ap + n + 1);
    std::vector<TileDesc> tiles;
    std::vector<int> tp;
    std::vector<long long> br;
    if (breaks != nullptr) br.assign(breaks, breaks + n_breaks + 1);
    build_tiles(H, G, T, RMAX, breaks ? &br : nullptr, tiles, breaks ? &tp : nullptr);
    if ((int)tiles.size() > cap) return fail(AMGB_EINVAL, "build_tiles: output capacity too small");
    for (size_t t = 0; t < tiles.size(); t++) { row0[t] = tiles[t].row0; nz0[t] = tiles[t].nz0; }
    if (tile_ptr != nullptr && breaks != nullptr)
        for (size_t w = 0; w < tp.size(); w++) tile_ptr[w] = tp[w];
    *n_tiles = (int32_t)tiles.size() - 1;
    return AMGB_OK;
}

// Dependency waves of a sequential sweep (host only, no CUDA): wave_of[k] (1-based) for list position k.
// The multi-GPU layer uses it to give every rank the same global wave structure.
extern "C" int amgb_wave_schedule(int32_t n, const int32_t *Ap, const int32_t *Aj, const int32_t *list, int64_t m,
                                  int32_t *wave_of, int32_t *n_waves)
{
    if (Ap == nullptr || wave_of == nullptr || n < 0 || m < 0) return fail(AMGB_EINVAL, "wave_schedule: bad arguments");
    std::vector<int> wwave((size_t)n, 0), rwave((size_t)n, 0);
    int maxw = 0;
    for (int64_t k = 0; k < m; k++) {
        const int i = list ? list[k] : (int)k;
        if (i < 0 || i >= n) return fail(AMGB_EINVAL, "wave_schedule: row index out of range");
        int wv = std::max(rwave[(size_t)i], wwave[(size_t)i]);
        for (int jj = Ap[i]; jj < Ap[i + 1]; jj++) {
            const int j = Aj[jj];
            if (j != i && j >= 0 && j < n) wv = std::max(wv, wwave[(size_t)j]);
        }
        wv += 1;
        wave_of[k] = wv;
        wwave[(size_t)i] = wv;
        for (int jj = Ap[i]; jj < Ap[i + 1]; jj++) {
            const int j = Aj[jj];
            if (j != i && j >= 0 && j < n) rwave[(size_t)j] = std::max(rwave[(size_t)j], wv);
        }
        maxw = std::max(maxw, wv);
    }
    if (n_waves) *n_waves = maxw;
    return AMGB_OK;
}

// ------------------------------------------------------------------------------------------
// C ABI (3): device kernels
// ------------------------------------------------------------------------------------------
// S = the current device's settings, *out = the lanes per row of a call (lanes = 0: from the mean row length)
static int resolve_lanes(Settings &S, int lanes, int32_t n_rows, const int32_t *Ap, cudaStream_t s, int *out)
{
    RET(current_settings(S));
    if (lanes == 0) {
        int nnz = 0;
        if (n_rows > 0) {
            CK(cudaMemcpyAsync(&nnz, Ap + n_rows, sizeof(int), cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        lanes = pick_lanes(S, nnz, n_rows);
    }
    if (lanes < 1 || lanes > 32 || (lanes & (lanes - 1))) return fail(AMGB_EINVAL, "lanes must be a power of two in 1..32");
    *out = lanes;
    return AMGB_OK;
}

extern "C" int64_t amgb_dev_partials_len(int32_t n_rows, int lanes)
{
    if (lanes <= 0) lanes = 32;
    return csr_grid(n_rows, lanes) + 1;
}

static CsrRowArgs mk_args(int n, int row0, const int *rows, const int *Ap, const int *Aj, const double *Ax,
                          const double *x, const double *b, double *y, double *r, double omega, double *parts)
{
    CsrRowArgs a;
    a.n = n; a.row0 = row0; a.rows = rows; a.Ap = Ap; a.Aj = Aj; a.Ax = Ax;
    a.x = x; a.b = b; a.y = y; a.r = r; a.omega = omega; a.partials = parts;
    return a;
}

extern "C" int amgb_dev_csr_spmv(int32_t n_rows, const int32_t *Ap, const int32_t *Aj, const double *Ax,
                                 const double *x, double *y, int lanes, void *stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    Settings S;
    RET(resolve_lanes(S, lanes, n_rows, Ap, s, &lanes));
    return launch_csr(S, OP_SPMV, lanes, mk_args(n_rows, 0, nullptr, Ap, Aj, Ax, x, nullptr, y, nullptr, 0.0, nullptr), s);
}

extern "C" int amgb_dev_csr_residual(int32_t n_rows, const int32_t *Ap, const int32_t *Aj, const double *Ax,
                                     const double *x, const double *b, double *r, double *partials,
                                     double *norm2_out, int lanes, void *stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    Settings S;
    RET(resolve_lanes(S, lanes, n_rows, Ap, s, &lanes));
    if ((partials == nullptr) != (norm2_out == nullptr))
        return fail(AMGB_EINVAL, "partials and norm2_out must be given together");
    RET(launch_csr(S, OP_RESID, lanes, mk_args(n_rows, 0, nullptr, Ap, Aj, Ax, x, b, r, nullptr, 0.0, partials), s));
    if (partials != nullptr) {
        reduce_partials_kernel<<<1, 1024, 0, s>>>(partials, (int)csr_grid(n_rows, lanes), norm2_out);
        CK(cudaGetLastError());
    }
    return AMGB_OK;
}

extern "C" int amgb_dev_csr_spmv_add(int32_t n_rows, const int32_t *Ap, const int32_t *Aj, const double *Ax,
                                     const double *xc, double *x, int lanes, void *stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    Settings S;
    RET(resolve_lanes(S, lanes, n_rows, Ap, s, &lanes));
    return launch_csr(S, OP_PADD, lanes, mk_args(n_rows, 0, nullptr, Ap, Aj, Ax, xc, nullptr, x, nullptr, 0.0, nullptr), s);
}

extern "C" int amgb_dev_csr_jacobi(int32_t n_rows, const int32_t *Ap, const int32_t *Aj, const double *Ax,
                                   const double *x_in, const double *b, double *x_out, double *r_out,
                                   double omega, int lanes, void *stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    if (x_in == x_out) return fail(AMGB_EINVAL, "jacobi: x_in and x_out must differ");
    Settings S;
    RET(resolve_lanes(S, lanes, n_rows, Ap, s, &lanes));
    return launch_csr(S, OP_JACOBI, lanes, mk_args(n_rows, 0, nullptr, Ap, Aj, Ax, x_in, b, x_out, r_out, omega, nullptr), s);
}

extern "C" int amgb_dev_csr_gs_wave(int32_t n, int32_t row0, const int32_t *rows, const int32_t *Ap,
                                    const int32_t *Aj, const double *Ax, double *x, const double *b,
                                    double omega, int lanes, void *stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    if (lanes == 0) lanes = 8;
    if (lanes < 1 || lanes > 32 || (lanes & (lanes - 1))) return fail(AMGB_EINVAL, "lanes must be a power of two in 1..32");
    Settings S;
    RET(current_settings(S));
    return launch_csr(S, OP_GS, lanes, mk_args(n, row0, rows, Ap, Aj, Ax, x, b, x, nullptr, omega, nullptr), s);
}

extern "C" int amgb_dev_dense_matvec(int32_t m, int32_t n, const double *M, const double *x, double *y,
                                     void *stream)
{
    if (m <= 0) return AMGB_OK;
    dense_matvec_kernel<<<(m + 3) / 4, 128, 0, (cudaStream_t)stream>>>(m, n, M, x, y);
    CK(cudaGetLastError());
    return AMGB_OK;
}

extern "C" int amgb_dev_gather(const double *in, const int32_t *idx, double *out, int64_t n, void *stream)
{
    if (n <= 0) return AMGB_OK;
    Settings S;
    RET(current_settings(S));
    gather_kernel<<<vec_grid(S, n), 256, 0, (cudaStream_t)stream>>>(in, idx, out, n);
    CK(cudaGetLastError());
    return AMGB_OK;
}

extern "C" int amgb_dev_fill(double *x, int64_t n, double v, void *stream)
{
    Settings S;
    RET(current_settings(S));
    return launch_fill(S, x, n, v, (cudaStream_t)stream);
}

// out_dev[0] = <x, y> (x == y: the squared 2-norm) with the engine's deterministic two-stage reduction;
// scratch: amgb_dev_reduce_len() doubles of device memory
extern "C" int64_t amgb_dev_reduce_len(void) { return kSumsqBlocks; }

extern "C" int amgb_dev_dot(const double *x, const double *y, int64_t n, double *scratch, double *out_dev, void *stream)
{
    if (x == nullptr || y == nullptr || scratch == nullptr || out_dev == nullptr) return fail(AMGB_EINVAL, "null pointer");
    if (n < 0) return fail(AMGB_EINVAL, "n < 0");
    cudaStream_t s = (cudaStream_t)stream;
    Settings S;
    RET(current_settings(S));
    dot_partials_kernel<<<sumsq_blocks(S), 256, 0, s>>>(x, y, n, scratch);
    CK(cudaGetLastError());
    reduce_partials_kernel<<<1, 1024, 0, s>>>(scratch, sumsq_blocks(S), out_dev);
    CK(cudaGetLastError());
    return AMGB_OK;
}

// y = a x + b y
extern "C" int amgb_dev_axpby(double a, const double *x, double b, double *y, int64_t n, void *stream)
{
    if (n <= 0) return AMGB_OK;
    if (x == nullptr || y == nullptr) return fail(AMGB_EINVAL, "null pointer");
    Settings S;
    RET(current_settings(S));
    axpby_kernel<<<vec_grid(S, n), 256, 0, (cudaStream_t)stream>>>(a, x, b, y, n);
    CK(cudaGetLastError());
    return AMGB_OK;
}

// block Jacobi sweep on the point-CSR expansion of a BSR operator (what the engine uploads): n_block_rows block rows
// of size bs, Dinv (n_block_rows, bs, bs) row-major, x_out != x_in
extern "C" int amgb_dev_block_jacobi(int32_t n_block_rows, int32_t bs, const int32_t *Ap, const int32_t *Aj,
                                     const double *Ax, const double *x_in, const double *b, const double *Dinv,
                                     double *x_out, double omega, int lanes, void *stream)
{
    if (x_in == x_out) return fail(AMGB_EINVAL, "block_jacobi: x_in and x_out must differ");
    if (lanes == 0) lanes = 8;
    if (lanes < 1 || lanes > 32 || (lanes & (lanes - 1))) return fail(AMGB_EINVAL, "lanes must be a power of two in 1..32");
    DevCsr A;
    A.Ap = const_cast<int *>(Ap); A.Aj = const_cast<int *>(Aj); A.Ax = const_cast<double *>(Ax);
    return dispatch_block_jacobi(bs, lanes, n_block_rows, A, x_in, b, Dinv, x_out, omega, (cudaStream_t)stream);
}
