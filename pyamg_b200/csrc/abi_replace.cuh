// abi_replace.cuh -- part of engine.cu's translation unit (included there): amgb_hierarchy_replace_level0, a new
// fine-level matrix under a resident hierarchy (MultilevelSolver.change_solve_matrix, pyamg/multilevel.py:320-337).
//
// Levels >= 1, the coarse solver, the zero-start copies, the AMLI buffers and the K-wide level blocks stay as they
// are.  Path 1 (same pattern, same smoother structure, same value stream) writes the new values into level 0's
// existing arrays; path 2 rebuilds level 0 as finalize_levels builds it (build_level), from the new matrix and the
// P_0 / R_0 already on the device.  Either way level 0 ends up as a fresh upload of the same levels would leave it.
#pragma once

// dst[s] = src[map[s]] (times scale when SCALE): refills a reordered copy of level 0's values from the values in
// source order.  map is the source entry of every slot of the copy (Level0Refresh).
template <bool SCALE>
__global__ void __launch_bounds__(256) refresh_slots_kernel(double *__restrict__ dst, const double *__restrict__ src,
                                                            const int *__restrict__ map, long long n, double scale)
{
    for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += (long long)gridDim.x * blockDim.x) {
        const double v = src[map[s]];
        dst[s] = SCALE ? scale * v : v;
    }
}

static int refresh_slots(const Settings &S, double *dst, const double *src, const int *map, long long n,
                         const double *scale, cudaStream_t s)
{
    if (n <= 0) return AMGB_OK;
    const unsigned grid = vec_grid(S, n);
    if (scale != nullptr) refresh_slots_kernel<true><<<grid, 256, 0, s>>>(dst, src, map, n, *scale);
    else refresh_slots_kernel<false><<<grid, 256, 0, s>>>(dst, src, map, n, 1.0);
    CK(cudaGetLastError());
    return AMGB_OK;
}

template <typename T>
static int download(std::vector<T> &v, const T *d, long long n)
{
    v.resize((size_t)n);
    if (n > 0) CK(cudaMemcpy(v.data(), d, sizeof(T) * (size_t)n, cudaMemcpyDeviceToHost));
    return AMGB_OK;
}

static int download_csr(const DevCsr &D, HostCsr &H)
{
    H.n_rows = D.n_rows;
    H.n_cols = D.n_cols;
    RET(download(H.Ap, (const int *)D.Ap, (long long)D.n_rows + 1));
    RET(download(H.Aj, (const int *)D.Aj, D.nnz));
    return download(H.Ax, (const double *)D.Ax, D.nnz);
}

// Everything of a smoother that build_level derives from the pattern and the descriptor's structure: equal
// structures on the same pattern give the same schedules, row lists and layout
static bool same_structure(const SmootherSpec &a, const SmootherSpec &b)
{
    return a.kind == b.kind && a.iterations == b.iterations && a.sweep == b.sweep && a.bs == b.bs &&
           a.has_list == b.has_list && a.list == b.list && a.list2 == b.list2 && a.f_iterations == b.f_iterations &&
           a.c_iterations == b.c_iterations && a.coef.size() == b.coef.size();
}

static void release_smoother(amgb_hierarchy *h, Smoother &s)
{
    h->release(s.ws.rows); h->release(s.Dinv); h->release(s.rows1); h->release(s.rows2);
    h->release_csr(s.ne_A); h->release_csr(s.ne_At);
    h->release(s.sz_Sj); h->release(s.sz_Sp); h->release(s.sz_Tp);
    h->release(s.res_wave_ptr); h->release(s.res_seq);
    s = Smoother();
}

// The slot maps of the column-sorted copy of level 0 (ne_A, the Schwarz copy) and of its transpose (ne_At): the same
// sort and transpose make_smoother applies, run on the entry indices
static int ensure_sorted_maps(amgb_hierarchy *h, const HostCsr &A)
{
    Level0Refresh &re = h->re0;
    if (re.map_sorted != nullptr) return AMGB_OK;
    HostCsr I = A, T;
    for (size_t k = 0; k < I.Ax.size(); k++) I.Ax[k] = (double)k;      // exact: nnz < 2^31
    sort_rows_by_column(I);
    transpose_csr(I, T);
    std::vector<int> m(I.Ax.size());
    for (size_t k = 0; k < m.size(); k++) m[k] = (int)I.Ax[k];
    RET(h->upload(&re.map_sorted, m.data(), (long long)m.size()));
    for (size_t k = 0; k < m.size(); k++) m[k] = (int)T.Ax[k];
    return h->upload(&re.map_T, m.data(), (long long)m.size());
}

// Path 1.  *done = false (nothing changed) when the new level 0 would be laid out or streamed differently.
static int refresh_level0(amgb_hierarchy *h, const HostLevel &H, cudaStream_t s, bool *done)
{
    *done = false;
    Level &L = h->levels[0];
    if (!same_structure(H.pre, h->spec0[0]) || !same_structure(H.post, h->spec0[1])) return AMGB_OK;
    if ((long long)H.A.Aj.size() != L.A.nnz) return AMGB_OK;
    std::vector<int> order, pos;
    if (h->order0 != nullptr) {
        RET(download(order, (const int *)h->order0, L.A.n_rows));
        RET(download(pos, (const int *)h->pos0, L.A.n_rows));
    }
    HostCsr B;                                          // the new operator in level-0 numbering
    if (!order.empty()) permute_csr(H.A, order.data(), pos.data(), B);
    const HostCsr &A = order.empty() ? H.A : B;
    Level0Refresh &re = h->re0;
    if (re.have_pattern) {
        if (H.A.Ap != re.Ap || H.A.Aj != re.Aj) return AMGB_OK;
    } else {                                            // first call: compare with what level 0 holds
        std::vector<int> Ap, Aj;
        RET(download(Ap, (const int *)L.A.Ap, (long long)L.A.n_rows + 1));
        RET(download(Aj, (const int *)L.A.Aj, L.A.nnz));
        if (A.Ap != Ap || A.Aj != Aj) return AMGB_OK;
        re.Ap = H.A.Ap;
        re.Aj = H.A.Aj;
        re.have_pattern = true;
    }
    ValueStream v;
    if (h->S.use_tiles) h->value_stream(A, L.A, h->S.use_value_codes, v);
    const int format = L.A.rcodes ? ValueStream::ROW : L.A.pairs ? ValueStream::PAIR
                     : L.A.codes ? ValueStream::VALUE : ValueStream::FP64;
    if (v.format != format) return AMGB_OK;
    *done = true;
    const long long nnz = L.A.nnz;
    CK(cudaMemcpyAsync(L.A.Ax, A.Ax.data(), sizeof(double) * (size_t)nnz, cudaMemcpyHostToDevice, s));
    // a table that grew gets a new block; codes and the padded pattern table keep theirs
    auto table = [&](auto *&dst, const auto &src) -> int {
        if ((int)src.size() > L.A.ndict) {
            h->release(dst);
            return h->upload(&dst, src.data(), (long long)src.size());
        }
        CK(cudaMemcpyAsync(dst, src.data(), sizeof(src[0]) * src.size(), cudaMemcpyHostToDevice, s));
        return AMGB_OK;
    };
    switch (format) {
    case ValueStream::ROW:
        CK(cudaMemcpyAsync(L.A.rcodes, v.codes.data(), (size_t)L.A.n_rows, cudaMemcpyHostToDevice, s));
        L.A.npatterns = (int)v.pats.size();
        v.pats.resize((size_t)kMaxCodes, RowPattern{});
        CK(cudaMemcpyAsync(L.A.patterns, v.pats.data(), sizeof(RowPattern) * v.pats.size(), cudaMemcpyHostToDevice, s));
        RET(table(L.A.pairs, v.pairs));
        L.A.ndict = (int)v.pairs.size();
        break;
    case ValueStream::PAIR:
        CK(cudaMemcpyAsync(L.A.codes, v.codes.data(), (size_t)nnz, cudaMemcpyHostToDevice, s));
        RET(table(L.A.pairs, v.pairs));
        L.A.ndict = (int)v.pairs.size();
        break;
    case ValueStream::VALUE:
        CK(cudaMemcpyAsync(L.A.codes, v.codes.data(), (size_t)nnz, cudaMemcpyHostToDevice, s));
        RET(table(L.A.dict, v.dict));
        L.A.ndict = (int)v.dict.size();
        break;
    }
    for (int k = 0; k < 2; k++) {
        Smoother &sm = k ? L.post : L.pre;
        const SmootherSpec &sp = k ? H.post : H.pre;
        sm.omega = sp.omega;
        sm.coef = sp.coef;
        if (sm.Dinv != nullptr && !sp.Dinv.empty())
            CK(cudaMemcpyAsync(sm.Dinv, sp.Dinv.data(), sizeof(double) * sp.Dinv.size(), cudaMemcpyHostToDevice, s));
        // the sorted copies exist only on unpermuted levels (make_smoother), so L.A.Ax is in source order
        if (sm.ne_A.Ax != nullptr) {
            RET(ensure_sorted_maps(h, H.A));
            RET(refresh_slots(h->S, sm.ne_A.Ax, L.A.Ax, re.map_sorted, nnz, nullptr, s));
        }
        if (sm.ne_At.Ax != nullptr)        // jacobi_ne keeps omega A^T (make_smoother)
            RET(refresh_slots(h->S, sm.ne_At.Ax, L.A.Ax, re.map_T, nnz, sp.kind == AMGB_SM_JACOBI_NE ? &sp.omega : nullptr, s));
    }
    CK(cudaStreamSynchronize(s));                       // the host arrays above die with this call
    return AMGB_OK;
}

// Path 2: level 0 rebuilt from the new matrix and smoothers; P_0's rows and R_0's columns follow its new numbering
static int rebuild_level0(amgb_hierarchy *h, HostLevel &H)
{
    Level &L = h->levels[0];
    const long long n = L.A.n_rows;
    std::vector<int> order, pos;
    if (h->order0 != nullptr) {
        RET(download(order, (const int *)h->order0, n));
        RET(download(pos, (const int *)h->pos0, n));
    }
    HostCsr Pd, Rd;
    RET(download_csr(L.P, Pd));
    RET(download_csr(L.R, Rd));
    if (order.empty()) {
        H.P = std::move(Pd);
        H.R = std::move(Rd);
    } else {                                            // back to the caller's level-0 numbering
        permute_csr(Pd, pos.data(), nullptr, H.P);
        permute_csr(Rd, nullptr, order.data(), H.R);
    }
    H.has_pr = true;
    const int old_lanes = L.A.lanes;
    h->release_csr(L.A);
    h->release_csr(L.P);
    h->release_csr(L.R);
    release_smoother(h, L.pre);
    release_smoother(h, L.post);
    h->release(h->order0);
    h->release(h->pos0);
    h->release(h->io_tmp);
    Level0Refresh &re = h->re0;
    h->release(re.map_sorted);
    h->release(re.map_T);
    re.Ap = H.A.Ap;                                     // the next same-pattern change compares with these
    re.Aj = H.A.Aj;
    re.have_pattern = true;
    LevelLayout Y;
    h->plan_layout(H, Y);
    RET(h->build_level(0, H, Y, nullptr));
    RET(h->resident_prepare(L, L.pre));
    RET(h->resident_prepare(L, L.post));
    // buffers finalize and the batched solves size from level 0's operator and smoothers
    if ((L.pre.kind == AMGB_SM_POLYNOMIAL || L.post.kind == AMGB_SM_POLYNOMIAL) && L.poly[0] == nullptr) {
        RET(h->dalloc(&L.poly[0], n + 2));
        RET(h->dalloc(&L.poly[1], n + 2));
        for (ManyWidth &mw : h->many)
            if (!mw.lv.empty()) {
                const long long k = 2LL << (&mw - h->many);          // widths 2, 4, 8
                RET(h->dalloc(&mw.lv[0].poly[0], n * k + 2));
                RET(h->dalloc(&mw.lv[0].poly[1], n * k + 2));
            }
    }
    const long long np = std::max<long long>(3 * h->partials_len(L.A), 1);
    if (np > h->n_partials) {
        h->release(h->partials);
        RET(h->dalloc(&h->partials, np));
        h->n_partials = np;
    }
    if (csr_grid(n, L.A.lanes) > csr_grid(n, old_lanes))
        for (int i = 0; i < 3; i++) {
            ManyWidth &mw = h->many[i];
            if (mw.lv.empty()) continue;
            h->release(mw.partials);
            RET(h->dalloc(&mw.partials, many_partials_len(h->S, L.A) * (2LL << i)));
        }
    return AMGB_OK;
}

// Captured launch sequences bake in level-0 pointers and scalars (omega): they are captured again on next use
static void drop_captures(amgb_hierarchy *h)
{
    for (int k = 0; k < 4; k++) {
        if (h->graph[k]) cudaGraphExecDestroy(h->graph[k]);
        if (h->graph_stop[k]) cudaGraphExecDestroy(h->graph_stop[k]);
        h->graph[k] = h->graph_stop[k] = nullptr;
        h->release(h->tail_prog[k].dev);
        h->tail_prog[k] = amgb_hierarchy::TailProg();
    }
    for (ManyWidth &mw : h->many)
        for (cudaGraphExec_t &g : mw.graph) {
            if (g) cudaGraphExecDestroy(g);
            g = nullptr;
        }
}

extern "C" int amgb_hierarchy_replace_level0(amgb_hierarchy *h, const amgb_matrix *A, const amgb_smoother *pre,
                                             const amgb_smoother *post, void *stream, int32_t *path)
{
    if (h == nullptr || path == nullptr) return fail(AMGB_EINVAL, "null argument");
    *path = 0;
    if (!h->finalized) return fail(AMGB_ESTATE, "hierarchy not finalized");
    if (h->levels.size() < 2) return fail(AMGB_ENOTIMPL, "one-level hierarchy: level 0 is the coarse level");
    HostLevel H;
    RET(to_host_csr(A, H.A, "A"));
    const Level &L = h->levels[0];
    if (H.A.n_rows != L.A.n_rows || H.A.n_cols != L.A.n_cols) return fail(AMGB_EINVAL, "A: shape differs from level 0");
    RET(copy_smoother(pre, H.A, H.pre));
    RET(copy_smoother(post, H.A, H.post));
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));              // no solve in flight may still read level 0
    const cudaStream_t s = stream ? (cudaStream_t)stream : h->stream;
    drop_captures(h);
    h->release_csr(h->At0);                            // A^H of the old matrix: the caller sets the new one
    bool done = false;
    int rc = refresh_level0(h, H, s, &done);
    if (rc == AMGB_OK && !done) rc = rebuild_level0(h, H);
    if (rc != AMGB_OK) {
        h->finalized = false;                          // level 0 may be half replaced: no solve may run on it
        return rc;
    }
    CK(cudaStreamSynchronize(h->stream));
    *path = done ? 1 : 2;
    return AMGB_OK;
}
