// multi_rhs_kernels.cuh -- K right-hand sides per pass over an operator (MultilevelSolver.solve_many, abi_many.cuh).
//
// A K-wide vector block is n x K row-major: column j of row i at v[i*K + j] (K = 2, 4, 8).  Every kernel reads
// each stored operator entry once and applies it to the K columns; a gather of x[c] is K/2 16-byte loads of one
// contiguous 8K-byte run, so at K = 4 one 32-byte sector per entry.
//
// Summation order.  Column j of a batched cycle must equal the single-vector cycle on that column, so every
// kernel keeps the lane -> entry assignment and the shuffle tree of the kernel `solve` launches for the same
// operator, with K accumulators per lane:
//   many_rows_kernel   lanes-per-row (csr_rows_kernel): G lanes per row, lane l takes entries l, l+G, ...
//   many_tile_kernel   one warp per host-built tile (csr_tile_kernel / csr_tile_flat_kernel): G lanes per row, or
//                      for the flat-gather operators (G == 0) g = the largest power of two with g * rows <= 32 per
//                      tile and the product rounded before the add (the flat kernel stores it to shared memory);
//                      a row longer than the tile bound is summed by the whole warp, as both tile kernels do.
//   many_block_jacobi_kernel, many_block_gs_kernel   G lanes per block row (block_jacobi_kernel, block_gs_kernel),
//                      then lane 0 applies the block's Dinv row-major.
// The operator is read straight from global memory (no TMA staging): at K = 8 the staged b / x_old slices alone
// would take RMAX * K * 8 B per warp and halve the resident warps.
//
// Epilogues as csr_kernels.cuh (OP_SPMV, OP_RESID + K per-column |r|^2 partials, OP_PADD, OP_JACOBI, OP_GS).
#pragma once
#include "tile_kernels.cuh"

namespace amgb {

struct ManyArgs {
    int n;                   // rows kernel: rows of this launch
    int row0;                // rows kernel: first row (rows == nullptr)
    const int *rows;         // rows kernel: explicit row list (Gauss-Seidel waves of an un-permuted level)
    const TileDesc *tiles;   // tile kernel: descriptors, tiles [tile_begin, tile_end)
    int tile_begin, tile_end;
    int G;                   // lanes per row (power of two); tile kernel: 0 = flat-gather split
    int T;                   // tile kernel: rows with more entries than this are summed by the whole warp
    const int *Ap;
    const int *Aj;
    const double *Ax;
    const double *x;         // n_cols x K
    const double *b;         // n_rows x K
    double *y;               // n_rows x K (OP_GS: == x)
    double omega;
    double *partials;        // OP_RESID: K per block (block-major), or nullptr
};

// K consecutive doubles (16-byte aligned: K is even and every block is a cudaMalloc allocation)
template <int K, bool NC>
__device__ __forceinline__ void ld_k(const double *p, double (&o)[K])
{
#ifdef AMGB_EMU
#pragma unroll
    for (int q = 0; q < K; q++) o[q] = p[q];
#else
#pragma unroll
    for (int q = 0; q < K; q += 2) {
        const double2 t = NC ? __ldg(reinterpret_cast<const double2 *>(p + q)) : *reinterpret_cast<const double2 *>(p + q);
        o[q] = t.x;
        o[q + 1] = t.y;
    }
#endif
}

// K block-wide sums (fixed order) -> out[0..K) by thread 0
template <int THREADS, int K>
__device__ __forceinline__ void block_sum_k(double (&v)[K], double *out)
{
    __shared__ double s_part[THREADS / 32][K];
#pragma unroll
    for (int q = 0; q < K; q++) v[q] = group_sum<32>(v[q]);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) {
#pragma unroll
        for (int q = 0; q < K; q++) s_part[w][q] = v[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int q = 0; q < K; q++) {
            double t = 0.0;
            for (int i = 0; i < THREADS / 32; i++) t += s_part[i][q];
            out[q] = t;
        }
    }
}

// one row group: g lanes (sub = lane in group) sum entries [jb, je) of `row`, then the fused epilogue.
// All 32 lanes of the warp call this with the same g (the shuffles are warp-wide).
template <int K, int OP>
__device__ __forceinline__ void many_row(const ManyArgs &a, bool active, int row, int jb, int je, int sub, int g,
                                         bool flat, double (&r2)[K])
{
    constexpr bool kNeedDiag = (OP == OP_JACOBI || OP == OP_GS);
    double sum[K];
#pragma unroll
    for (int q = 0; q < K; q++) sum[q] = 0.0;
    double diag = 0.0;
    int jd = -1;
    for (int jj = jb + sub; jj < je; jj += g) {
        const int c = __ldg(a.Aj + jj);
        const double v = __ldg(a.Ax + jj);
        if (kNeedDiag && c == row) {    // later duplicates overwrite
            diag = v;
            jd = jj;
            continue;
        }
        double xv[K];
        ld_k<K, OP != OP_GS>(a.x + (size_t)c * K, xv);
        if (flat) {
#pragma unroll
            for (int q = 0; q < K; q++) sum[q] += __dmul_rn(v, xv[q]);
        } else {
#pragma unroll
            for (int q = 0; q < K; q++) sum[q] += v * xv[q];
        }
    }
    for (int o = g >> 1; o > 0; o >>= 1) {
#pragma unroll
        for (int q = 0; q < K; q++) sum[q] += __shfl_xor_sync(0xffffffffu, sum[q], o);
        if (kNeedDiag) {
            const int jo = __shfl_xor_sync(0xffffffffu, jd, o);
            const double dv = __shfl_xor_sync(0xffffffffu, diag, o);
            if (jo > jd) { jd = jo; diag = dv; }
        }
    }
    if (!active || sub != 0) return;
    const size_t base = (size_t)row * K;
    if (OP == OP_SPMV) {
#pragma unroll
        for (int q = 0; q < K; q++) a.y[base + q] = sum[q];
    } else if (OP == OP_RESID) {
        double bv[K];
        ld_k<K, true>(a.b + base, bv);
#pragma unroll
        for (int q = 0; q < K; q++) {
            const double r = bv[q] - sum[q];
            a.y[base + q] = r;
            r2[q] += r * r;
        }
    } else if (OP == OP_PADD) {
#pragma unroll
        for (int q = 0; q < K; q++) a.y[base + q] += sum[q];
    } else if (OP == OP_JACOBI) {
        double bv[K], xv[K];
        ld_k<K, true>(a.b + base, bv);
        ld_k<K, true>(a.x + base, xv);
#pragma unroll
        for (int q = 0; q < K; q++) {
            double xn = xv[q];
            if (diag != 0.0) xn = (1.0 - a.omega) * xv[q] + a.omega * ((bv[q] - sum[q]) / diag);
            a.y[base + q] = xn;
        }
    } else if (diag != 0.0) {   // OP_GS
        double bv[K];
        ld_k<K, true>(a.b + base, bv);
#pragma unroll
        for (int q = 0; q < K; q++) {
            const double gs = (bv[q] - sum[q]) / diag;
            a.y[base + q] = (a.omega == 1.0) ? gs : a.omega * gs + (1.0 - a.omega) * a.y[base + q];
        }
    }
}

template <int K, int OP>
__global__ void __launch_bounds__(kCsrThreads) many_rows_kernel(const ManyArgs a)
{
    const int g = a.G;
    const int lane = threadIdx.x & (g - 1);
    const long long k = ((long long)blockIdx.x * kCsrThreads + threadIdx.x) / g;
    const bool active = k < a.n;
    int row = 0, start = 0, end = 0;
    if (active) {
        row = a.rows ? a.rows[k] : a.row0 + (int)k;
        start = a.Ap[row];
        end = a.Ap[row + 1];
    }
    double r2[K];
#pragma unroll
    for (int q = 0; q < K; q++) r2[q] = 0.0;
    many_row<K, OP>(a, active, row, start, end, lane, g, false, r2);
    if (OP == OP_RESID && a.partials != nullptr) block_sum_k<kCsrThreads, K>(r2, a.partials + (size_t)blockIdx.x * K);
}

constexpr int kManyTileWarps = 8;

template <int K, int OP>
__global__ void __launch_bounds__(kManyTileWarps * 32) many_tile_kernel(const ManyArgs a)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nwarps = gridDim.x * kManyTileWarps;
    double r2[K];
#pragma unroll
    for (int q = 0; q < K; q++) r2[q] = 0.0;
    for (int t = a.tile_begin + blockIdx.x * kManyTileWarps + warp; t < a.tile_end; t += nwarps) {
        const TileDesc d0 = a.tiles[t], d1 = a.tiles[t + 1];
        const int nrows = d1.row0 - d0.row0;
        if (d1.nz0 - d0.nz0 > a.T) {        // a single row longer than a tile: the whole warp
            many_row<K, OP>(a, true, d0.row0, d0.nz0, d1.nz0, lane, 32, false, r2);
            continue;
        }
        const bool flat = a.G == 0;
        int g = a.G;
        if (flat) {
            g = 32;
            while (g > 1 && g * nrows > 32) g >>= 1;
        }
        const int rpp = 32 / g, sub = lane & (g - 1), grp = lane / g;
        for (int rbase = 0; rbase < nrows; rbase += rpp) {
            const int lr = rbase + grp;
            const bool active = lr < nrows;
            const int row = d0.row0 + lr;
            int jb = 0, je = 0;
            if (active) {
                jb = a.Ap[row];
                je = a.Ap[row + 1];
            }
            many_row<K, OP>(a, active, row, jb, je, sub, g, flat, r2);
        }
    }
    if (OP == OP_RESID && a.partials != nullptr)
        block_sum_k<kManyTileWarps * 32, K>(r2, a.partials + (size_t)blockIdx.x * K);
}

// block Jacobi (engine.cu block_jacobi_kernel) on K columns: G lanes per block row
template <int K, int BS>
__global__ void __launch_bounds__(kCsrThreads) many_block_jacobi_kernel(int G, int nb, const int *__restrict__ Ap,
                                                                        const int *__restrict__ Aj,
                                                                        const double *__restrict__ Ax,
                                                                        const double *__restrict__ x,
                                                                        const double *__restrict__ b,
                                                                        const double *__restrict__ Dinv,
                                                                        double *__restrict__ y, double omega)
{
    const int lane = threadIdx.x & (G - 1);
    const long long I = ((long long)blockIdx.x * kCsrThreads + threadIdx.x) / G;
    const bool active = I < nb;
    const int Ib = active ? (int)I : -1;
    double rs[BS][K];
#pragma unroll
    for (int k = 0; k < BS; k++) {
        double sum[K];
#pragma unroll
        for (int q = 0; q < K; q++) sum[q] = 0.0;
        if (active) {
            const int row = (int)I * BS + k;
            const int s = Ap[row], e = Ap[row + 1];
            for (int jj = s + lane; jj < e; jj += G) {
                const int c = ld_stream_i32(Aj + jj);
                const double v = ld_stream_f64(Ax + jj);
                if (c / BS != Ib) {
                    double xv[K];
                    ld_k<K, true>(x + (size_t)c * K, xv);
#pragma unroll
                    for (int q = 0; q < K; q++) sum[q] += v * xv[q];
                }
            }
        }
        for (int o = G >> 1; o > 0; o >>= 1) {
#pragma unroll
            for (int q = 0; q < K; q++) sum[q] += __shfl_xor_sync(0xffffffffu, sum[q], o);
        }
#pragma unroll
        for (int q = 0; q < K; q++) rs[k][q] = sum[q];
    }
    if (active && lane == 0) {
        const size_t base = (size_t)I * BS;
#pragma unroll
        for (int k = 0; k < BS; k++)
#pragma unroll
            for (int q = 0; q < K; q++) rs[k][q] = b[(base + k) * K + q] - rs[k][q];
#pragma unroll
        for (int k = 0; k < BS; k++) {
#pragma unroll
            for (int q = 0; q < K; q++) {
                double v = 0.0;
#pragma unroll
                for (int c = 0; c < BS; c++) v += Dinv[base * BS + (size_t)k * BS + c] * rs[c][q];
                y[(base + k) * K + q] = (1.0 - omega) * x[(base + k) * K + q] + omega * v;
            }
        }
    }
}

// one wave of block Gauss-Seidel (engine.cu block_gs_kernel) on K columns: G lanes per listed block row, which
// read the current iterate and write x_I = Dinv_I (b_I - rsum) in place (no block of a wave reads another block
// of the same wave)
template <int K, int BS>
__global__ void __launch_bounds__(kCsrThreads) many_block_gs_kernel(int G, int nrows, const int *__restrict__ brows,
                                                                    const int *__restrict__ Ap,
                                                                    const int *__restrict__ Aj,
                                                                    const double *__restrict__ Ax, double *x,
                                                                    const double *__restrict__ b,
                                                                    const double *__restrict__ Dinv)
{
    const int lane = threadIdx.x & (G - 1);
    const long long i = ((long long)blockIdx.x * kCsrThreads + threadIdx.x) / G;
    const bool active = i < nrows;
    const int I = active ? brows[i] : 0;
    double rs[BS][K];
#pragma unroll
    for (int k = 0; k < BS; k++) {
        double sum[K];
#pragma unroll
        for (int q = 0; q < K; q++) sum[q] = 0.0;
        if (active) {
            const int row = I * BS + k;
            const int s = Ap[row], e = Ap[row + 1];
            for (int jj = s + lane; jj < e; jj += G) {
                const int c = ld_stream_i32(Aj + jj);
                const double v = ld_stream_f64(Ax + jj);
                if (c / BS != I) {
                    double xv[K];
                    ld_k<K, false>(x + (size_t)c * K, xv);      // plain loads: x is written by this launch
#pragma unroll
                    for (int q = 0; q < K; q++) sum[q] += v * xv[q];
                }
            }
        }
        for (int o = G >> 1; o > 0; o >>= 1) {
#pragma unroll
            for (int q = 0; q < K; q++) sum[q] += __shfl_xor_sync(0xffffffffu, sum[q], o);
        }
#pragma unroll
        for (int q = 0; q < K; q++) rs[k][q] = sum[q];
    }
    if (active && lane == 0) {
        const size_t base = (size_t)I * BS;
#pragma unroll
        for (int k = 0; k < BS; k++)
#pragma unroll
            for (int q = 0; q < K; q++) rs[k][q] = b[(base + k) * K + q] - rs[k][q];
#pragma unroll
        for (int k = 0; k < BS; k++) {
#pragma unroll
            for (int q = 0; q < K; q++) {
                double v = 0.0;
#pragma unroll
                for (int c = 0; c < BS; c++) v += Dinv[base * BS + (size_t)k * BS + c] * rs[c][q];
                x[(base + k) * K + q] = v;
            }
        }
    }
}

// one conflict wave of gauss_seidel_ne / gauss_seidel_nr (kaczmarz_kernel) on K columns: G lanes per listed row of M
// with the single kernel's lane -> entry map and shuffle tree, K inner products per lane, then K deltas and K scatter
// updates per entry.  The rows of a wave share no column, so no two groups update the same entry of v; v is read
// and written by this launch (plain loads).
//   NE: delta = (b_i - sum) * Dinv_i * omega ;  v_j += m_ij * delta                          (v = x)
//   NR: delta = sum * (Dinv_i * omega)       ;  x_i += delta ; v_j -= delta * m_ij           (v = r, xout = x)
template <int K, int G, bool NR>
__global__ void __launch_bounds__(kCsrThreads) many_kaczmarz_kernel(int nrows, const int *__restrict__ rows,
                                                                    const int *__restrict__ Mp,
                                                                    const int *__restrict__ Mj,
                                                                    const double *__restrict__ Mx, double *v,
                                                                    const double *__restrict__ b,
                                                                    const double *__restrict__ Dinv, double omega,
                                                                    double *xout)
{
    const int lane = threadIdx.x & (G - 1);
    const long long k = ((long long)blockIdx.x * kCsrThreads + threadIdx.x) / G;
    const bool active = k < nrows;
    int row = 0, start = 0, end = 0;
    if (active) {
        row = rows[k];
        start = Mp[row];
        end = Mp[row + 1];
    }
    double sum[K];
#pragma unroll
    for (int q = 0; q < K; q++) sum[q] = 0.0;
    for (int jj = start + lane; jj < end; jj += G) {
        const double m = Mx[jj];
        double vv[K];
        ld_k<K, false>(v + (size_t)Mj[jj] * K, vv);
#pragma unroll
        for (int q = 0; q < K; q++) sum[q] += m * vv[q];
    }
#pragma unroll
    for (int q = 0; q < K; q++) sum[q] = group_sum<G>(sum[q]);
    if (!active) return;                           // (after the shuffles: inactive groups took part in them)
    double delta[K];
    if (NR) {
        const double s = Dinv[row] * omega;
#pragma unroll
        for (int q = 0; q < K; q++) delta[q] = sum[q] * s;
        if (lane == 0) {
#pragma unroll
            for (int q = 0; q < K; q++) xout[(size_t)row * K + q] += delta[q];
        }
        for (int jj = start + lane; jj < end; jj += G) {
            const double m = Mx[jj];
            double *p = v + (size_t)Mj[jj] * K;
#pragma unroll
            for (int q = 0; q < K; q++) p[q] -= delta[q] * m;
        }
    } else {
        double bv[K];
        ld_k<K, true>(b + (size_t)row * K, bv);
        const double d = Dinv[row];
#pragma unroll
        for (int q = 0; q < K; q++) delta[q] = (bv[q] - sum[q]) * d * omega;
        for (int jj = start + lane; jj < end; jj += G) {
            const double m = Mx[jj];
            double *p = v + (size_t)Mj[jj] * K;
#pragma unroll
            for (int q = 0; q < K; q++) p[q] += m * delta[q];
        }
    }
}

// one wave of multiplicative overlapping Schwarz (schwarz_kernel) on K columns: one warp per subdomain, every lane
// forms whole local rows sequentially in the single kernel's order -- r_j -= a x_j over the row, + b_j; then
// u_j += T_qc rsum_cj in ascending c -- for the K columns at once; all reads of x precede the updates (two warp
// barriers).  Shared memory: 2 * max_m * K doubles per warp, local row q's K values contiguous.
template <int K>
__global__ void __launch_bounds__(kSchwarzWarps * 32) many_schwarz_kernel(int ndom, const int *__restrict__ doms,
                                                                         const int *__restrict__ Sp,
                                                                         const int *__restrict__ Sj,
                                                                         const long long *__restrict__ Tp,
                                                                         const double *__restrict__ Tx,
                                                                         const int *__restrict__ Ap,
                                                                         const int *__restrict__ Aj,
                                                                         const double *__restrict__ Ax, double *x,
                                                                         const double *__restrict__ b, int max_m)
{
    extern __shared__ __align__(16) unsigned char many_schwarz_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double *rsum = reinterpret_cast<double *>(many_schwarz_smem) + (size_t)warp * 2 * max_m * K;
    double *upd = rsum + (size_t)max_m * K;
    const int k = blockIdx.x * kSchwarzWarps + warp;
    const bool active = k < ndom;             // whole warps are active or not: the warp barriers below stay converged
    int s0 = 0, m = 0;
    long long t0 = 0;
    if (active) {
        const int d = doms[k];
        s0 = Sp[d];
        m = Sp[d + 1] - s0;
        t0 = Tp[d];
    }
    for (int q = lane; q < m; q += 32) {
        const int row = Sj[s0 + q];
        double r[K];
#pragma unroll
        for (int j = 0; j < K; j++) r[j] = 0.0;
        for (int jj = Ap[row]; jj < Ap[row + 1]; jj++) {
            const double a = Ax[jj];
            double xv[K];
            ld_k<K, false>(x + (size_t)Aj[jj] * K, xv);
#pragma unroll
            for (int j = 0; j < K; j++) r[j] -= a * xv[j];
        }
        double bv[K];
        ld_k<K, true>(b + (size_t)row * K, bv);
#pragma unroll
        for (int j = 0; j < K; j++) rsum[(size_t)q * K + j] = r[j] + bv[j];
    }
    __syncwarp();
    for (int q = lane; q < m; q += 32) {
        double u[K];
#pragma unroll
        for (int j = 0; j < K; j++) u[j] = 0.0;
        const double *Trow = Tx + t0 + (long long)q * m;
        for (int c = 0; c < m; c++) {
            const double t = Trow[c];
#pragma unroll
            for (int j = 0; j < K; j++) u[j] += t * rsum[(size_t)c * K + j];
        }
#pragma unroll
        for (int j = 0; j < K; j++) upd[(size_t)q * K + j] = u[j];
    }
    __syncwarp();
    for (int q = lane; q < m; q += 32) {
        double *p = x + (size_t)Sj[s0 + q] * K;
#pragma unroll
        for (int j = 0; j < K; j++) p[j] += upd[(size_t)q * K + j];
    }
}

// y[i*K + q] *= s[i] (mul_kernel with row i's scale broadcast to its K entries): jacobi_ne's delta = (b - A x) Dinv
template <int K>
__global__ void __launch_bounds__(256) many_mul_rows_kernel(double *__restrict__ y, const double *__restrict__ s,
                                                            long long nk)
{
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nk; i += (long long)gridDim.x * 256)
        y[i] = y[i] * s[i / K];
}

// y = M x for the dense coarse operator (dense_matvec_kernel): one warp per row, lane-strided columns
template <int K>
__global__ void many_dense_matvec_kernel(int m, int n, const double *__restrict__ M, const double *__restrict__ x,
                                         double *__restrict__ y)
{
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int l = threadIdx.x & 31;
    if (w >= m) return;
    double s[K];
#pragma unroll
    for (int q = 0; q < K; q++) s[q] = 0.0;
    for (int j = l; j < n; j += 32) {
        const double mv = M[(size_t)w * n + j];
        double xv[K];
        ld_k<K, true>(x + (size_t)j * K, xv);
#pragma unroll
        for (int q = 0; q < K; q++) s[q] += mv * xv[q];
    }
#pragma unroll
    for (int q = 0; q < K; q++) s[q] = group_sum<32>(s[q]);
    if (l == 0) {
#pragma unroll
        for (int q = 0; q < K; q++) y[(size_t)w * K + q] = s[q];
    }
}

// dst (n x K) = columns [0, w) of src (row pitch ld, rows taken through `order` when it is set), zero columns
// [w, K): the caller's column slice into the level-0 block (wave-major order on a permuted level)
template <int K>
__global__ void many_pack_kernel(const double *__restrict__ src, long long ld, int w, const int *__restrict__ order,
                                 double *__restrict__ dst, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n * K; i += stride) {
        const long long row = i / K;
        const int q = (int)(i % K);
        const long long from = order ? order[row] : row;
        dst[i] = q < w ? src[from * ld + q] : 0.0;
    }
}

// columns [q0, q1) of src (n x K) -> dst (row pitch ld), row `row` going to order[row] when `order` is set
template <int K>
__global__ void many_unpack_kernel(const double *__restrict__ src, const int *__restrict__ order, double *__restrict__ dst,
                                   long long ld, int q0, int q1, long long n)
{
    const int w = q1 - q0;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n * w; i += stride) {
        const long long row = i / w;
        const int q = q0 + (int)(i % w);
        const long long to = order ? order[row] : row;
        dst[to * ld + q] = src[row * K + q];
    }
}

// partials[blk*K + q] = sum of x[i*K+q]^2 over block blk's grid-stride share (fixed grid: deterministic)
template <int K>
__global__ void __launch_bounds__(256) many_sumsq_kernel(const double *__restrict__ x, long long n,
                                                         double *__restrict__ partials)
{
    double t[K];
#pragma unroll
    for (int q = 0; q < K; q++) t[q] = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double v[K];
        ld_k<K, true>(x + (size_t)i * K, v);
#pragma unroll
        for (int q = 0; q < K; q++) t[q] += v[q] * v[q];
    }
    block_sum_k<256, K>(t, partials + (size_t)blockIdx.x * K);
}

// partials[blk*K + q] = sum of x[i*K+q]*y[i*K+q] over block blk's grid-stride share: dot_partials_kernel per column
// (same grid, same order), so after many_reduce_kernel column q's dot is dev_dot's on that column bit for bit
template <int K>
__global__ void __launch_bounds__(256) many_dot_kernel(const double *__restrict__ x, const double *__restrict__ y,
                                                       long long n, double *__restrict__ partials)
{
    double t[K];
#pragma unroll
    for (int q = 0; q < K; q++) t[q] = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double xv[K], yv[K];
        ld_k<K, true>(x + (size_t)i * K, xv);
        ld_k<K, true>(y + (size_t)i * K, yv);
#pragma unroll
        for (int q = 0; q < K; q++) t[q] += xv[q] * yv[q];
    }
    block_sum_k<256, K>(t, partials + (size_t)blockIdx.x * K);
}

// per-column coefficients of many_axpby_kernel (K <= 8), passed by value; columns outside `active` are not written
struct ManyAxpby {
    double a[8], b[8];
    unsigned active;
};

// y[i*K+q] = a[q]*x[i*K+q] + b[q]*y[i*K+q] for the active columns: axpby_kernel's expression, so nvcc contracts it
// to the same DFMA form and each column equals dev_axpby on it
template <int K>
__global__ void __launch_bounds__(256) many_axpby_kernel(const ManyAxpby c, const double *__restrict__ x,
                                                         double *__restrict__ y, long long n)
{
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double xv[K], yv[K];
        ld_k<K, true>(x + (size_t)i * K, xv);
        ld_k<K, false>(y + (size_t)i * K, yv);
#pragma unroll
        for (int q = 0; q < K; q++)
            if (c.active & (1u << q)) y[(size_t)i * K + q] = c.a[q] * xv[q] + c.b[q] * yv[q];
    }
}

// out[q] = sum over m partials[i*K + q] in a fixed order (one block)
template <int K>
__global__ void __launch_bounds__(1024) many_reduce_kernel(const double *partials, int m, double *out)
{
    double t[K];
#pragma unroll
    for (int q = 0; q < K; q++) t[q] = 0.0;
    for (int i = threadIdx.x; i < m; i += 1024) {
#pragma unroll
        for (int q = 0; q < K; q++) t[q] += partials[(size_t)i * K + q];
    }
    block_sum_k<1024, K>(t, out);
}

// ---------------------------------------------------------------------------------------------
// Householder GMRES / flexible GMRES on K columns (abi_many_gmres.cuh).  Each kernel is its single-vector twin in
// csr_kernels.cuh applied per column, with the same expression (so the same contraction) per entry; the writing
// kernels leave every column outside `active` untouched.
// ---------------------------------------------------------------------------------------------
// one value per column (K <= 8), passed by value
struct ManyScalars {
    double v[8];
    unsigned active;
};

// v_q = (I - 2 w_q w_q^T) e_k = (-2 w[k,q]) w_q + e_k                   (hh_unit_reflect_kernel per column)
template <int K>
__global__ void __launch_bounds__(256) many_hh_unit_reflect_kernel(double *__restrict__ v, const double *__restrict__ w,
                                                                   long long k, unsigned active, long long n)
{
    double f[K];
#pragma unroll
    for (int q = 0; q < K; q++) f[q] = -2.0 * w[(size_t)k * K + q];
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double wv[K];
        ld_k<K, true>(w + (size_t)i * K, wv);
#pragma unroll
        for (int q = 0; q < K; q++) {
            if (!(active & (1u << q))) continue;
            double t = f[q] * wv[q];
            if (i == k) t = t + 1.0;
            v[(size_t)i * K + q] = t;
        }
    }
}

// w_q = [0 ... 0, v[k1,q] + alpha_q, v[k1+1,q], ...] on the columns in alpha.active (hh_make_w_kernel per column).
// w may alias v: every entry is read and written by the same thread.
template <int K>
__global__ void __launch_bounds__(256) many_hh_make_w_kernel(double *w, const double *v, long long k1,
                                                             const ManyScalars alpha, long long n)
{
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
#pragma unroll
        for (int q = 0; q < K; q++) {
            if (!(alpha.active & (1u << q))) continue;
            double t = (i < k1) ? 0.0 : v[(size_t)i * K + q];
            if (i == k1) t += alpha.v[q];
            w[(size_t)i * K + q] = t;
        }
    }
}

// y_q = y_q / d_q (div_kernel per column)
template <int K>
__global__ void __launch_bounds__(256) many_div_kernel(double *__restrict__ y, const ManyScalars d, long long n)
{
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
#pragma unroll
        for (int q = 0; q < K; q++)
            if (d.active & (1u << q)) y[(size_t)i * K + q] = y[(size_t)i * K + q] / d.v[q];
    }
}

// y_q = a_q x_q (scale_kernel per column: the first term of FGMRES's Z y; never reads y)
template <int K>
__global__ void __launch_bounds__(256) many_scale_kernel(double *__restrict__ y, const ManyScalars a,
                                                         const double *__restrict__ x, long long n)
{
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
#pragma unroll
        for (int q = 0; q < K; q++)
            if (a.active & (1u << q)) y[(size_t)i * K + q] = a.v[q] * x[(size_t)i * K + q];
    }
}

// partials[blk*K + q] = sum of x[i,q]^2 over i >= start of block blk's grid-stride share (sumsq_from_partials_kernel
// per column: same grid, same order; reduced by many_reduce_kernel)
template <int K>
__global__ void __launch_bounds__(256) many_sumsq_from_kernel(const double *__restrict__ x, long long start, long long n,
                                                              double *__restrict__ partials)
{
    double t[K];
#pragma unroll
    for (int q = 0; q < K; q++) t[q] = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        if (i < start) continue;
        double v[K];
        ld_k<K, true>(x + (size_t)i * K, v);
#pragma unroll
        for (int q = 0; q < K; q++) t[q] += v[q] * v[q];
    }
    block_sum_k<256, K>(t, partials + (size_t)blockIdx.x * K);
}

// y_q += sign * (num[q] / den[0]) * x_q with num read from device memory (axpy_ratio_kernel per column): a
// reflection's inner product never leaves the device
template <int K>
__global__ void __launch_bounds__(256) many_axpy_ratio_kernel(double *__restrict__ y, const double *__restrict__ x,
                                                              const double *num, const double *den, double sign,
                                                              unsigned active, long long n)
{
    double a[K];
#pragma unroll
    for (int q = 0; q < K; q++) a[q] = sign * (num[q] / den[0]);
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double xv[K];
        ld_k<K, true>(x + (size_t)i * K, xv);
#pragma unroll
        for (int q = 0; q < K; q++)
            if (active & (1u << q)) y[(size_t)i * K + q] += a[q] * xv[q];
    }
}

// x[i, q] += v_q on the active columns (add_at_kernel per column; one thread, the columns unrolled so that the
// by-value coefficients stay in registers)
template <int K>
__global__ void many_add_at_kernel(double *x, long long i, const ManyScalars v)
{
#pragma unroll
    for (int q = 0; q < K; q++)
        if (v.active & (1u << q)) x[(size_t)i * K + q] += v.v[q];
}

// One fused MGS step on K columns (mgs_step_kernel per column, abi_many_gmres.cuh): v_q -= c_q * vprev_q on the
// columns in `active` with c_q = coef[q] from the previous step's many_reduce_kernel, then the block partials of
// <vk_q, v_q> (dots) and <v_q, v_q> (sq), block-major as many_dot_kernel.  The expressions are mgs_step_kernel's, so
// nvcc contracts them to the same DFMAs: fma(-c, p, x) for the update, fma(a, b, t) for the sums.  Columns outside
// `active` are not written; their partials are formed and never read.
template <int K>
__global__ void __launch_bounds__(256) many_mgs_step_kernel(double *__restrict__ v, const double *__restrict__ vprev,
                                                            const double *__restrict__ coef,
                                                            const double *__restrict__ vk, unsigned active, long long n,
                                                            double *__restrict__ dots, double *__restrict__ sq)
{
    double c[K], td[K], ts[K];
#pragma unroll
    for (int q = 0; q < K; q++) {
        c[q] = vprev != nullptr ? coef[q] : 0.0;
        td[q] = 0.0;
        ts[q] = 0.0;
    }
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double x[K];
        ld_k<K, false>(v + (size_t)i * K, x);
        if (vprev != nullptr) {
            double p[K];
            ld_k<K, true>(vprev + (size_t)i * K, p);
#pragma unroll
            for (int q = 0; q < K; q++) {
                if (!(active & (1u << q))) continue;
                x[q] = x[q] - c[q] * p[q];
                v[(size_t)i * K + q] = x[q];
            }
        }
        if (dots != nullptr) {
            double w[K];
            ld_k<K, true>(vk + (size_t)i * K, w);
#pragma unroll
            for (int q = 0; q < K; q++) td[q] += w[q] * x[q];
        }
        if (sq != nullptr) {
#pragma unroll
            for (int q = 0; q < K; q++) ts[q] += x[q] * x[q];
        }
    }
    if (dots != nullptr) block_sum_k<256, K>(td, dots + (size_t)blockIdx.x * K);
    if (sq != nullptr) {
        __syncthreads();                           // block_sum_k's shared partials are reused
        block_sum_k<256, K>(ts, sq + (size_t)blockIdx.x * K);
    }
}

// y_q = x_q * (1.0 / h_q), h_q = sqrt(nsq[q]), when h_q != 0, else y_q = x_q, on the columns in `active`
// (mgs_scale_kernel per column)
template <int K>
__global__ void __launch_bounds__(256) many_mgs_scale_kernel(double *__restrict__ y, const double *__restrict__ x,
                                                             const double *nsq, unsigned active, long long n)
{
    double h[K], r[K];
#pragma unroll
    for (int q = 0; q < K; q++) {
        h[q] = sqrt(nsq[q]);
        r[q] = 1.0 / h[q];
    }
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double xv[K];
        ld_k<K, true>(x + (size_t)i * K, xv);
#pragma unroll
        for (int q = 0; q < K; q++)
            if (active & (1u << q)) y[(size_t)i * K + q] = h[q] != 0.0 ? xv[q] * r[q] : xv[q];
    }
}

// stagnation test per column: partials[blk*K + q] = max |u[i,q] / x[i,q]| over x[i,q] != 0, -1 if the share has
// none (maxratio_partials_kernel per column)
template <int K>
__global__ void __launch_bounds__(256) many_maxratio_kernel(const double *__restrict__ u, const double *__restrict__ x,
                                                            long long n, double *__restrict__ partials)
{
    __shared__ double s_max[8][K];
    double t[K];
#pragma unroll
    for (int q = 0; q < K; q++) t[q] = -1.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double uv[K], xv[K];
        ld_k<K, true>(u + (size_t)i * K, uv);
        ld_k<K, true>(x + (size_t)i * K, xv);
#pragma unroll
        for (int q = 0; q < K; q++)
            if (xv[q] != 0.0) t[q] = fmax(t[q], fabs(uv[q] / xv[q]));
    }
#pragma unroll
    for (int q = 0; q < K; q++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t[q] = fmax(t[q], __shfl_xor_sync(0xffffffffu, t[q], o));
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int q = 0; q < K; q++) s_max[threadIdx.x >> 5][q] = t[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int q = 0; q < K; q++) {
            for (int i = 1; i < 8; i++) t[q] = fmax(t[q], s_max[i][q]);
            partials[(size_t)blockIdx.x * K + q] = t[q];
        }
    }
}

// out[q] = max over m partials[i*K + q] (reduce_max_kernel per column; one block)
template <int K>
__global__ void __launch_bounds__(1024) many_reduce_max_kernel(const double *partials, int m, double *out)
{
    __shared__ double s_max[32][K];
    double t[K];
#pragma unroll
    for (int q = 0; q < K; q++) t[q] = -1.0;
    for (int i = threadIdx.x; i < m; i += 1024) {
#pragma unroll
        for (int q = 0; q < K; q++) t[q] = fmax(t[q], partials[(size_t)i * K + q]);
    }
#pragma unroll
    for (int q = 0; q < K; q++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t[q] = fmax(t[q], __shfl_xor_sync(0xffffffffu, t[q], o));
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int q = 0; q < K; q++) s_max[threadIdx.x >> 5][q] = t[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int q = 0; q < K; q++) {
            for (int i = 1; i < 32; i++) t[q] = fmax(t[q], s_max[i][q]);
            out[q] = t[q];
        }
    }
}

}  // namespace amgb
