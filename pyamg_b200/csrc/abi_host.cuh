// abi_host.cuh -- part of engine.cu's translation unit (included there): the reference-FFI-shaped host entry
// points (amgb_host_*), amgb_host_relax and the SciPy-bit-identical Galerkin SpGEMM driver.  Not a stand-alone header.
#pragma once

// ------------------------------------------------------------------------------------------
// C ABI (2): reference-FFI-shaped host entry points.  Upload, run the same kernels, download.
// ------------------------------------------------------------------------------------------
namespace {
struct Scratch {   // RAII device scratch for the host-shaped calls
    std::vector<void *> ptrs;
    ~Scratch() { for (void *p : ptrs) cudaFree(p); }
    template <typename T>
    int up(T **d, const T *h, long long n)
    {
        void *q = nullptr;
        CK(cudaMalloc(&q, (size_t)std::max<long long>(n, 1) * sizeof(T)));
        ptrs.push_back(q);
        if (n > 0 && h != nullptr) CK(cudaMemcpy(q, h, (size_t)n * sizeof(T), cudaMemcpyHostToDevice));
        *d = (T *)q;
        return AMGB_OK;
    }
};

int check_csr_host(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size, const double *Ax,
                   int Ax_size, int x_size, int b_size, int vals_per_entry)
{
    if (Ap == nullptr || Ap_size < 1) return fail(AMGB_EINVAL, "Ap missing");
    if (Aj_size > 0 && (Aj == nullptr || Ax == nullptr)) return fail(AMGB_EINVAL, "Aj/Ax missing");
    if ((long long)Aj_size * vals_per_entry != (long long)Ax_size) return fail(AMGB_EINVAL, "Aj/Ax size mismatch");
    if (Ap[Ap_size - 1] != Aj_size) return fail(AMGB_EINVAL, "Ap[-1] != len(Aj)");
    if (x_size != b_size) return fail(AMGB_EINVAL, "x and b sizes differ");
    return AMGB_OK;
}

// rows visited by `for (i = start; i != stop; i += step)`
int range_rows(int start, int stop, int step, int n, std::vector<int> &rows)
{
    rows.clear();
    if (step == 0) return fail(AMGB_EINVAL, "row_step == 0");
    if ((stop - start) % step != 0) return fail(AMGB_EINVAL, "row range never terminates");
    if ((stop - start) / step < 0) return fail(AMGB_EINVAL, "row range never terminates");
    for (int i = start; i != stop; i += step) {
        if (i < 0 || i >= n) return fail(AMGB_EINVAL, "row index out of range");
        rows.push_back(i);
    }
    return AMGB_OK;
}
}  // namespace

extern "C" int amgb_host_jacobi(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                                int b_size, double *temp, int temp_size, int32_t row_start,
                                int32_t row_stop, int32_t row_step, const double *omega, int omega_size)
{
    RET(check_csr_host(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x_size, b_size, 1));
    const int n = Ap_size - 1;
    if (x_size != n || temp_size < n || omega == nullptr || omega_size < 1)
        return fail(AMGB_EINVAL, "jacobi: bad vector sizes");
    std::vector<int> rows;
    RET(range_rows(row_start, row_stop, row_step, n, rows));
    if (rows.empty()) return AMGB_OK;
    Scratch sc;
    int *dAp, *dAj, *drows;
    double *dAx, *dx, *db, *dy;
    RET(sc.up(&dAp, Ap, Ap_size)); RET(sc.up(&dAj, Aj, Aj_size)); RET(sc.up(&dAx, Ax, Ax_size));
    RET(sc.up(&dx, (const double *)x, n)); RET(sc.up(&db, b, n)); RET(sc.up(&dy, (const double *)x, n));
    RET(sc.up(&drows, rows.data(), (long long)rows.size()));
    Settings S;
    RET(current_settings(S));
    const int lanes = pick_lanes(S, Aj_size, n);
    RET(launch_csr(S, OP_JACOBI, lanes, mk_args((int)rows.size(), 0, drows, dAp, dAj, dAx, dx, db, dy, nullptr, omega[0], nullptr), 0));
    CK(cudaDeviceSynchronize());
    for (int i : rows) temp[i] = x[i];                      // relaxation.h:325-327
    CK(cudaMemcpy(x, dy, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost));
    return AMGB_OK;
}

static int host_gs_common(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size, const double *Ax,
                          int Ax_size, double *x, int x_size, const double *b, int b_size,
                          const std::vector<int> &list, double omega = 1.0)
{
    RET(check_csr_host(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x_size, b_size, 1));
    const int n = Ap_size - 1;
    if (x_size != n) return fail(AMGB_EINVAL, "gauss_seidel: bad vector sizes");
    if (list.empty()) return AMGB_OK;
    HostCsr H;
    H.n_rows = H.n_cols = n;
    H.Ap.assign(Ap, Ap + Ap_size);
    H.Aj.assign(Aj, Aj + Aj_size);
    for (int c : H.Aj) if (c < 0 || c >= n) return fail(AMGB_EINVAL, "column index out of range");
    std::vector<int> rows;
    std::vector<long long> ptr;
    build_waves(H, list.data(), (long long)list.size(), rows, ptr);
    Scratch sc;
    int *dAp, *dAj, *drows;
    double *dAx, *dx, *db;
    RET(sc.up(&dAp, Ap, Ap_size)); RET(sc.up(&dAj, Aj, Aj_size)); RET(sc.up(&dAx, Ax, Ax_size));
    RET(sc.up(&dx, (const double *)x, n)); RET(sc.up(&db, b, n));
    RET(sc.up(&drows, rows.data(), (long long)rows.size()));
    Settings S;
    RET(current_settings(S));
    const int lanes = pick_lanes(S, Aj_size, n);
    for (size_t w = 0; w + 1 < ptr.size(); w++)
        RET(launch_csr(S, OP_GS, lanes, mk_args((int)(ptr[w + 1] - ptr[w]), 0, drows + ptr[w], dAp, dAj, dAx, dx, db, dx, nullptr, omega, nullptr), 0));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(x, dx, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost));
    return AMGB_OK;
}

extern "C" int amgb_host_gauss_seidel(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                      const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                                      int b_size, int32_t row_start, int32_t row_stop, int32_t row_step)
{
    if (Ap == nullptr || Ap_size < 1) return fail(AMGB_EINVAL, "Ap missing");
    std::vector<int> list;
    RET(range_rows(row_start, row_stop, row_step, Ap_size - 1, list));
    return host_gs_common(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x, x_size, b, b_size, list);
}

extern "C" int amgb_host_sor_gauss_seidel(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                          const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                                          int b_size, int32_t row_start, int32_t row_stop, int32_t row_step,
                                          double omega)
{
    if (Ap == nullptr || Ap_size < 1) return fail(AMGB_EINVAL, "Ap missing");
    std::vector<int> list;
    RET(range_rows(row_start, row_stop, row_step, Ap_size - 1, list));
    return host_gs_common(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x, x_size, b, b_size, list, omega);
}

extern "C" int amgb_host_gauss_seidel_indexed(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                              const double *Ax, int Ax_size, double *x, int x_size,
                                              const double *b, int b_size, const int32_t *Id, int Id_size,
                                              int32_t row_start, int32_t row_stop, int32_t row_step)
{
    if (Ap == nullptr || Ap_size < 1) return fail(AMGB_EINVAL, "Ap missing");
    std::vector<int> pos, list;
    RET(range_rows(row_start, row_stop, row_step, Id_size, pos));
    for (int k : pos) {
        if (Id[k] < 0 || Id[k] >= Ap_size - 1) return fail(AMGB_EINVAL, "row index out of range");
        list.push_back(Id[k]);
    }
    return host_gs_common(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x, x_size, b, b_size, list);
}

extern "C" int amgb_host_bsr_jacobi(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                    const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                                    int b_size, double *temp, int temp_size, int32_t row_start,
                                    int32_t row_stop, int32_t row_step, int32_t blocksize,
                                    const double *omega, int omega_size)
{
    if (blocksize < 1) return fail(AMGB_EINVAL, "blocksize < 1");
    RET(check_csr_host(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x_size, b_size, blocksize * blocksize));
    const int nb = Ap_size - 1, n = nb * blocksize;
    if (x_size != n || temp_size < n || omega == nullptr || omega_size < 1)
        return fail(AMGB_EINVAL, "bsr_jacobi: bad vector sizes");
    std::vector<int> brows;
    RET(range_rows(row_start, row_stop, row_step, nb, brows));
    if (brows.empty()) return AMGB_OK;
    amgb_matrix M;
    M.n_rows = M.n_cols = n; M.block_r = M.block_c = blocksize; M.nnz_blocks = Aj_size;
    M.indptr = Ap; M.indices = Aj; M.data = Ax;
    HostCsr H;
    RET(to_host_csr(&M, H, "A"));
    std::vector<int> rows;
    for (int I : brows) for (int k = 0; k < blocksize; k++) rows.push_back(I * blocksize + k);
    Scratch sc;
    int *dAp, *dAj, *drows;
    double *dAx, *dx, *db, *dy;
    RET(sc.up(&dAp, H.Ap.data(), (long long)H.Ap.size())); RET(sc.up(&dAj, H.Aj.data(), (long long)H.Aj.size()));
    RET(sc.up(&dAx, H.Ax.data(), (long long)H.Ax.size()));
    RET(sc.up(&dx, (const double *)x, n)); RET(sc.up(&db, b, n)); RET(sc.up(&dy, (const double *)x, n));
    RET(sc.up(&drows, rows.data(), (long long)rows.size()));
    Settings S;
    RET(current_settings(S));
    const int lanes = pick_lanes(S, (long long)H.Aj.size(), n);
    RET(launch_csr(S, OP_JACOBI, lanes, mk_args((int)rows.size(), 0, drows, dAp, dAj, dAx, dx, db, dy, nullptr, omega[0], nullptr), 0));
    CK(cudaDeviceSynchronize());
    for (int i = 0; i < (int)rows.size(); i++) temp[i] = x[i];   // relaxation.h:506-508
    CK(cudaMemcpy(x, dy, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost));
    return AMGB_OK;
}

extern "C" int amgb_host_block_jacobi(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                      const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                                      int b_size, const double *Tx, int Tx_size, double *temp, int temp_size,
                                      int32_t row_start, int32_t row_stop, int32_t row_step,
                                      const double *omega, int omega_size, int32_t blocksize)
{
    if (blocksize < 1 || blocksize > 8) return fail(AMGB_ENOTIMPL, "block_jacobi: blocksize must be 1..8");
    RET(check_csr_host(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x_size, b_size, blocksize * blocksize));
    const int nb = Ap_size - 1, n = nb * blocksize;
    if (x_size != n || temp_size < n || omega == nullptr || omega_size < 1 || Tx == nullptr ||
        Tx_size != nb * blocksize * blocksize)
        return fail(AMGB_EINVAL, "block_jacobi: bad vector sizes");
    if (!(row_start == 0 && row_stop == nb && row_step == 1))
        return fail(AMGB_ENOTIMPL, "block_jacobi: only the full forward range (what relaxation.py:483-484 passes)");
    if (nb == 0) return AMGB_OK;
    amgb_matrix M;
    M.n_rows = M.n_cols = n; M.block_r = M.block_c = blocksize; M.nnz_blocks = Aj_size;
    M.indptr = Ap; M.indices = Aj; M.data = Ax;
    HostCsr H;
    RET(to_host_csr(&M, H, "A"));
    Scratch sc;
    DevCsr D;
    double *dx, *db, *dy, *dD;
    RET(sc.up(&D.Ap, H.Ap.data(), (long long)H.Ap.size())); RET(sc.up(&D.Aj, H.Aj.data(), (long long)H.Aj.size()));
    RET(sc.up(&D.Ax, H.Ax.data(), (long long)H.Ax.size()));
    RET(sc.up(&dx, (const double *)x, n)); RET(sc.up(&db, b, n)); RET(sc.up(&dy, (const double *)x, n));
    RET(sc.up(&dD, Tx, Tx_size));
    D.n_rows = D.n_cols = n;
    Settings S;
    RET(current_settings(S));
    const int lanes = pick_lanes(S, (long long)H.Aj.size(), n);
    RET(dispatch_block_jacobi(blocksize, lanes, nb, D, dx, db, dD, dy, omega[0], 0));
    CK(cudaDeviceSynchronize());
    std::memcpy(temp, x, sizeof(double) * (size_t)n);           // relaxation.h:1043-1045
    CK(cudaMemcpy(x, dy, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost));
    return AMGB_OK;
}

extern "C" int amgb_host_relax(const amgb_matrix *A, const amgb_smoother *sm, double *x, const double *b)
{
    if (A == nullptr || sm == nullptr || x == nullptr || b == nullptr) return fail(AMGB_EINVAL, "null argument");
    RET(validate_matrix(A, "A"));
    const int n = A->n_rows;
    if (n == 0) return AMGB_OK;
    // a two-level hierarchy whose transfer operators are empty: level 0 carries the operator and the smoother
    // through exactly the upload path of a real hierarchy (wave-major permutation, tiles, row lists)
    amgb_hierarchy *h = nullptr;
    RET(amgb_hierarchy_create(0, &h));
    struct Guard { amgb_hierarchy *h; ~Guard() { amgb_hierarchy_destroy(h); } } guard{h};
    std::vector<int32_t> p_ptr((size_t)n + 1, 0), one_ptr(2, 0);
    amgb_matrix P = {n, 1, 1, 1, 0, p_ptr.data(), nullptr, nullptr};
    amgb_matrix R = {1, n, 1, 1, 0, one_ptr.data(), nullptr, nullptr};
    amgb_matrix C = {1, 1, 1, 1, 0, one_ptr.data(), nullptr, nullptr};
    amgb_smoother none = {};
    none.kind = AMGB_SM_NONE;
    RET(amgb_hierarchy_add_level(h, A, &P, &R, sm, &none));
    RET(amgb_hierarchy_add_level(h, &C, nullptr, nullptr, nullptr, nullptr));
    RET(amgb_hierarchy_set_coarse_pinv(h, 1, nullptr, 1));
    RET(amgb_hierarchy_finalize(h, nullptr));
    h->launches = 0;
    RET(load_level0(h, b, x, cudaMemcpyHostToDevice));
    Level &L0 = h->levels[0];
    h->cur_level = 0;
    RET(h->smooth(L0, L0.pre));
    RET(store_level0(h, x, cudaMemcpyDeviceToHost));
    CK(cudaStreamSynchronize(h->stream));
    return AMGB_OK;
}

extern "C" int amgb_host_jacobi_indexed(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                        const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                                        int b_size, const int32_t *indices, int indices_size, const double *omega,
                                        int omega_size)
{
    RET(check_csr_host(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x_size, b_size, 1));
    const int n = Ap_size - 1;
    if (x_size != n || omega == nullptr || omega_size < 1) return fail(AMGB_EINVAL, "jacobi_indexed: bad vector sizes");
    if (indices_size < 0 || (indices_size > 0 && indices == nullptr)) return fail(AMGB_EINVAL, "jacobi_indexed: null row list");
    if (indices_size == 0 || n == 0) return AMGB_OK;
    amgb_matrix A = {n, n, 1, 1, Aj_size, Ap, Aj, Ax};
    amgb_smoother sm = {};
    sm.kind = AMGB_SM_JACOBI_INDEXED;
    sm.iterations = 1;
    sm.omega = omega[0];
    sm.indices = indices;
    sm.n_indices = indices_size;
    return amgb_host_relax(&A, &sm, x, b);
}

extern "C" int amgb_host_block_gauss_seidel(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                            const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                                            int b_size, const double *Tx, int Tx_size, int32_t row_start,
                                            int32_t row_stop, int32_t row_step, int32_t blocksize)
{
    if (blocksize < 1 || blocksize > 8) return fail(AMGB_ENOTIMPL, "block_gauss_seidel: blocksize must be 1..8");
    RET(check_csr_host(Ap, Ap_size, Aj, Aj_size, Ax, Ax_size, x_size, b_size, blocksize * blocksize));
    const int nb = Ap_size - 1, n = nb * blocksize;
    if (x_size != n || Tx == nullptr || (long long)Tx_size != (long long)n * blocksize)
        return fail(AMGB_EINVAL, "block_gauss_seidel: bad vector sizes");
    if (nb == 0) return AMGB_OK;
    amgb_smoother sm = {};
    sm.kind = AMGB_SM_BLOCK_GAUSS_SEIDEL;
    sm.iterations = 1;
    sm.blocksize = blocksize;
    sm.Dinv = Tx;
    if (row_start == 0 && row_stop == nb && row_step == 1) sm.sweep = AMGB_SWEEP_FORWARD;
    else if (row_start == nb - 1 && row_stop == -1 && row_step == -1) sm.sweep = AMGB_SWEEP_BACKWARD;
    else return fail(AMGB_ENOTIMPL, "block_gauss_seidel: only the full forward / backward block-row ranges");
    amgb_matrix A = {n, n, blocksize, blocksize, Aj_size, Ap, Aj, Ax};
    return amgb_host_relax(&A, &sm, x, b);
}

// ------------------------------------------------------------------------------------------
// C = A B as scipy.sparse._sparsetools.csr_matmat computes it (spgemm.cuh): the Galerkin product of the setup phase
// ------------------------------------------------------------------------------------------
template <int CAP, int THREADS>
static int launch_spgemm(SpgemmArgs a, cudaStream_t s)
{
    if (a.n_rows <= 0) return AMGB_OK;
    constexpr size_t smem = spgemm_smem_bytes<CAP>();
    static std::atomic<bool> attr_done[kMaxDevices];
    RET(optin_smem((const void *)spgemm_row_kernel<CAP, THREADS>, smem, attr_done));
    spgemm_row_kernel<CAP, THREADS><<<(unsigned)a.n_rows, THREADS, smem, s>>>(a);
    CK(cudaGetLastError());
    return AMGB_OK;
}

extern "C" void amgb_free(void *p) { free(p); }

extern "C" int amgb_host_csr_matmat(const amgb_matrix *A, const amgb_matrix *B, int32_t **Cp_out, int32_t **Cj_out,
                                    double **Cx_out, int64_t *nnz_out)
{
    if (Cp_out == nullptr || Cj_out == nullptr || Cx_out == nullptr || nnz_out == nullptr)
        return fail(AMGB_EINVAL, "null output");
    *Cp_out = nullptr; *Cj_out = nullptr; *Cx_out = nullptr; *nnz_out = 0;
    RET(validate_matrix(A, "A"));
    RET(validate_matrix(B, "B"));
    if (A->block_r != 1 || A->block_c != 1 || B->block_r != 1 || B->block_c != 1)
        return fail(AMGB_ENOTIMPL, "csr_matmat: CSR operands only (bsr_matmat is not on the GPU path)");
    if (A->n_cols != B->n_rows) return fail(AMGB_EINVAL, "dimension mismatch");       // scipy: ValueError
    const int n = A->n_rows;
    for (int64_t k = 0; k < A->nnz_blocks; k++)
        if (A->indices[k] < 0 || A->indices[k] >= A->n_cols) return fail(AMGB_EINVAL, "A: column index out of range");
    for (int64_t k = 0; k < B->nnz_blocks; k++)
        if (B->indices[k] < 0 || B->indices[k] >= B->n_cols) return fail(AMGB_EINVAL, "B: column index out of range");
    // bins by the work of a row: products (and entries of A_i, which index the offset table)
    std::vector<int> bins[3];
    static const int kCap[3] = {256, 2048, 8192};
    for (int i = 0; i < n; i++) {
        long long prod = 0;
        const int na = A->indptr[i + 1] - A->indptr[i];
        if (na < 0) return fail(AMGB_EINVAL, "A: indptr not monotone");
        for (int jj = A->indptr[i]; jj < A->indptr[i + 1]; jj++) {
            const int j = A->indices[jj];
            prod += B->indptr[j + 1] - B->indptr[j];
        }
        const long long need = std::max<long long>(prod, na);
        int b = 0;
        while (b < 3 && need > kCap[b]) b++;
        if (b == 3) return fail(AMGB_ENOTIMPL, "csr_matmat: a row with more than 8192 products");
        bins[b].push_back(i);
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return fail(AMGB_ECUDA, "no CUDA device");
    Scratch sc;
    SpgemmArgs a;
    int *dAp, *dAj, *dBp, *dBj, *d_rows[3], *d_nnz, *dCp, *dCj;
    double *dAx, *dBx, *dCx;
    RET(sc.up(&dAp, A->indptr, (long long)n + 1)); RET(sc.up(&dAj, A->indices, A->nnz_blocks));
    RET(sc.up(&dAx, A->data, A->nnz_blocks));
    RET(sc.up(&dBp, B->indptr, (long long)B->n_rows + 1)); RET(sc.up(&dBj, B->indices, B->nnz_blocks));
    RET(sc.up(&dBx, B->data, B->nnz_blocks));
    for (int b = 0; b < 3; b++) RET(sc.up(&d_rows[b], bins[b].data(), (long long)bins[b].size()));
    RET(sc.up(&d_nnz, (const int *)nullptr, (long long)n));
    a.Ap = dAp; a.Aj = dAj; a.Ax = dAx; a.Bp = dBp; a.Bj = dBj; a.Bx = dBx;
    a.row_nnz = d_nnz; a.Cp = nullptr; a.Cj = nullptr; a.Cx = nullptr;
    auto pass = [&](int fill) -> int {
        a.fill = fill;
        a.rows = d_rows[0]; a.n_rows = (int)bins[0].size();
        RET((launch_spgemm<256, 32>(a, 0)));
        a.rows = d_rows[1]; a.n_rows = (int)bins[1].size();
        RET((launch_spgemm<2048, 128>(a, 0)));
        a.rows = d_rows[2]; a.n_rows = (int)bins[2].size();
        RET((launch_spgemm<8192, 256>(a, 0)));
        CK(cudaDeviceSynchronize());
        return AMGB_OK;
    };
    RET(pass(0));
    std::vector<int> row_nnz((size_t)n);
    if (n > 0) CK(cudaMemcpy(row_nnz.data(), d_nnz, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost));
    int32_t *Cp = (int32_t *)malloc(sizeof(int32_t) * ((size_t)n + 1));
    if (Cp == nullptr) return fail(AMGB_ECUDA, "out of host memory");
    long long run = 0;
    Cp[0] = 0;
    for (int i = 0; i < n; i++) {
        run += row_nnz[(size_t)i];
        if (run > 2147483647LL) { free(Cp); return fail(AMGB_EINVAL, "csr_matmat: nnz exceeds int32 (reference index type)"); }
        Cp[i + 1] = (int32_t)run;
    }
    int32_t *Cj = (int32_t *)malloc(sizeof(int32_t) * (size_t)std::max<long long>(run, 1));
    double *Cx = (double *)malloc(sizeof(double) * (size_t)std::max<long long>(run, 1));
    struct OutGuard { int32_t *p, *j; double *x; bool keep; ~OutGuard() { if (!keep) { free(p); free(j); free(x); } } }
        og{Cp, Cj, Cx, false};
    if (Cj == nullptr || Cx == nullptr) return fail(AMGB_ECUDA, "out of host memory");
    RET(sc.up(&dCp, (const int *)Cp, (long long)n + 1));
    RET(sc.up(&dCj, (const int *)nullptr, run));
    RET(sc.up(&dCx, (const double *)nullptr, run));
    a.Cp = dCp; a.Cj = dCj; a.Cx = dCx;
    RET(pass(1));
    if (run > 0) {
        CK(cudaMemcpy(Cj, dCj, sizeof(int32_t) * (size_t)run, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(Cx, dCx, sizeof(double) * (size_t)run, cudaMemcpyDeviceToHost));
    }
    og.keep = true;
    *Cp_out = Cp; *Cj_out = Cj; *Cx_out = Cx; *nnz_out = run;
    return AMGB_OK;
}

extern "C" int amgb_host_matvec(const amgb_matrix *A, const double *x, double *y)
{
    HostCsr H;
    RET(to_host_csr(A, H, "A"));
    if (x == nullptr || y == nullptr) return fail(AMGB_EINVAL, "null vector");
    Scratch sc;
    int *dAp, *dAj;
    double *dAx, *dx, *dy;
    RET(sc.up(&dAp, H.Ap.data(), (long long)H.Ap.size())); RET(sc.up(&dAj, H.Aj.data(), (long long)H.Aj.size()));
    RET(sc.up(&dAx, H.Ax.data(), (long long)H.Ax.size()));
    RET(sc.up(&dx, x, H.n_cols)); RET(sc.up(&dy, (const double *)nullptr, H.n_rows));
    Settings S;
    RET(current_settings(S));
    const int lanes = pick_lanes(S, (long long)H.Aj.size(), H.n_rows);
    RET(launch_csr(S, OP_SPMV, lanes, mk_args(H.n_rows, 0, nullptr, dAp, dAj, dAx, dx, nullptr, dy, nullptr, 0.0, nullptr), 0));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(y, dy, sizeof(double) * (size_t)H.n_rows, cudaMemcpyDeviceToHost));
    return AMGB_OK;
}


// ---- device vertex colouring (SURVEY.md 8(f)-4) ----------------------------------------------------------------
// The reference's 'MIS' colouring (pyamg/graph.py:84-126 -> amg_core vertex_coloring_mis, graph.h:218-235) of the
// graph of a structurally symmetric CSR pattern, computed on the device as a wavefront of first-fit decisions
// (coloring.cuh).  Host arrays in, host colours out.  rounds_out (nullable): rounds the wavefront needed.
// More than 256 colours: AMGB_ENOTIMPL (callers fall back to the host routine).
extern "C" int amgb_host_vertex_coloring_mis(int32_t n, const int32_t *Ap, const int32_t *Aj, int32_t *colors,
                                             int32_t *n_colors, int32_t *rounds_out)
{
    if (n < 0 || Ap == nullptr || colors == nullptr || n_colors == nullptr) return fail(AMGB_EINVAL, "null pointer");
    *n_colors = 0;
    if (rounds_out) *rounds_out = 0;
    if (n == 0) return AMGB_OK;
    const long long nnz = Ap[n];
    if (nnz < 0 || (nnz > 0 && Aj == nullptr)) return fail(AMGB_EINVAL, "Aj missing");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return fail(AMGB_ECUDA, "no CUDA device");
    Scratch sc;
    int *dAp, *dAj, *dcol, *dflag;
    unsigned long long *drem;
    RET(sc.up(&dAp, Ap, (long long)n + 1));
    RET(sc.up(&dAj, Aj, nnz));
    RET(sc.up(&dcol, (const int *)nullptr, (long long)n));
    RET(sc.up(&dflag, (const int *)nullptr, 1));
    RET(sc.up(&drem, (const unsigned long long *)nullptr, 1));
    CK(cudaMemset(dcol, 0xFF, sizeof(int) * (size_t)n));             // -1: uncoloured
    CK(cudaMemset(dflag, 0, sizeof(int)));
    cudaDeviceProp prop;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaGetDeviceProperties(&prop, dev));
    const int grid = (int)std::min<long long>(((long long)n + 255) / 256, (long long)prop.multiProcessorCount * 8);
    int rounds = 0;
    const int kBatch = 8;                                            // rounds between two looks at the counter
    for (;;) {
        unsigned long long rem = 0;
        for (int b = 0; b < kBatch; b++) {
            CK(cudaMemsetAsync(drem, 0, sizeof(unsigned long long), 0));
            amgb::mis_color_round_kernel<<<grid, 256>>>(n, dAp, dAj, dcol, drem, dflag);
            CK(cudaGetLastError());
            rounds++;
        }
        CK(cudaMemcpy(&rem, drem, sizeof rem, cudaMemcpyDeviceToHost));
        if (rem == 0) break;
        if (rounds > 4 * n + 64) return fail(AMGB_ESTATE, "vertex colouring did not terminate (pattern not symmetric?)");
    }
    int over = 0;
    CK(cudaMemcpy(&over, dflag, sizeof over, cudaMemcpyDeviceToHost));
    if (over) return fail(AMGB_ENOTIMPL, "vertex colouring needs more than 256 colours");
    CK(cudaMemcpy(colors, dcol, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost));
    int k = 0;
    for (int i = 0; i < n; i++) k = std::max(k, colors[i] + 1);
    *n_colors = k;
    if (rounds_out) *rounds_out = rounds;
    return AMGB_OK;
}
