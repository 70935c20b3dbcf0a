// csr_kernels.cuh -- sm_90a CUDA kernels for the AMG solve-phase hot path (CSR operators).
//
// One kernel family, "G lanes per row": a group of G consecutive lanes (G = 2..32, chosen
// per operator from its mean row length) owns one row, strides over the row's (col,val)
// pairs with coalesced streaming loads, gathers x through the read-only/L1 path, and folds
// the partial sums with warp shuffles.  The epilogue is a template parameter so that every
// step of the V-cycle is ONE pass over its operator:
//
//   OP_SPMV    y_i  = sum_j a_ij x_j                          (restriction  b_c = R r;  SciPy csr_matvec,
//                                                              reference call site pyamg/multilevel.py:614)
//   OP_RESID   r_i  = b_i - sum_j a_ij x_j  [+ |r|^2 partials] (multilevel.py:612, :545/:567 with the norm fused)
//   OP_PADD    x_i += sum_j p_ij xc_j                          (multilevel.py:660, correction fused into the SpMV)
//   OP_JACOBI  x'_i = (1-w) x_i + w (b_i - sum_{j!=i} a_ij x_j)/a_ii ; optional r_i = b_i - (A x)_i
//                                                              (pyamg/amg_core/relaxation.h:309-346; the Jacobi sweep
//                                                              fused with the residual SpMV: one pass, two outputs)
//   OP_GS      x_i  = w (b_i - sum_{j!=i} a_ij x_j)/a_ii + (1-w) x_i  in place, over an independent set of rows
//                                                              (relaxation.h:48-76 / :736-768 executed wave by wave)
//
// Reference quirks honoured (SURVEY.md appendix): the diagonal is found by col==row (indices
// may be unsorted), the LAST stored duplicate of the diagonal wins, a zero diagonal leaves the
// row untouched.
//
// Roofline: all of these are HBM-bound (0.17 flop/byte); algorithmic bytes per launch are
// 12*nnz + 4*(n+1) + {16,24,24,32(+8),24(+4 indexed)}*n  (SURVEY.md 8(d)).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace amgb {

enum CsrOp { OP_SPMV = 0, OP_RESID = 1, OP_PADD = 2, OP_JACOBI = 3, OP_GS = 4 };

struct CsrRowArgs {
    int n;                 // rows handled by this launch
    int row0;              // first row (contiguous mode, rows == nullptr)
    const int *rows;       // explicit row list (indexed mode) or nullptr
    const int *Ap;
    const int *Aj;
    const double *Ax;
    const double *x;       // gathered vector (for OP_GS this aliases y)
    const double *b;
    double *y;             // output: y / r / x (PADD, GS in place) / x' (JACOBI)
    double *r;             // OP_JACOBI: optional residual by-product (nullptr = skip)
    double omega;
    double *partials;      // OP_RESID / OP_JACOBI(r): optional per-block sum of r_i^2 (nullptr = skip)
};

// streaming loads for the operator arrays: read once, keep them out of L1 so the x gathers own it
__device__ __forceinline__ int ld_stream_i32(const int *p)
{
#ifdef AMGB_EMU      // host-side emulation build (tests/emu): same logic, plain load
    return *p;
#else
    int v;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
#endif
}
__device__ __forceinline__ double ld_stream_f64(const double *p)
{
#ifdef AMGB_EMU
    return *p;
#else
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
#endif
}

// Programmatic dependent launch (sm_90+): a kernel launched with the programmatic-stream-serialization
// attribute may start while its predecessor in the stream is still running; it must not touch anything
// the predecessor produces before pdl_wait().  Without the attribute both are no-ops.
__device__ __forceinline__ void pdl_launch_dependents()
{
#ifndef AMGB_EMU
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}
__device__ __forceinline__ void pdl_wait()
{
#ifndef AMGB_EMU
    asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}

template <int G>
__device__ __forceinline__ double group_sum(double v)
{
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, G);
    return v;
}

// block-wide sum of one double per thread -> thread 0 (fixed order: deterministic)
template <int THREADS>
__device__ __forceinline__ double block_sum(double v)
{
    __shared__ double s_part[THREADS / 32];
    v = group_sum<32>(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) s_part[w] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < THREADS / 32; i++) t += s_part[i];
    }
    return t;
}

constexpr int kCsrThreads = 256;

template <int G, int OP, bool INDEXED>
__global__ void __launch_bounds__(kCsrThreads) csr_rows_kernel(const CsrRowArgs a)
{
    constexpr bool kNeedDiag = (OP == OP_JACOBI || OP == OP_GS);
    const int lane = threadIdx.x & (G - 1);
    const long long k = ((long long)blockIdx.x * kCsrThreads + threadIdx.x) / G;
    const bool active = k < a.n;
    double r2 = 0.0;  // this thread's contribution to |r|^2
    // PDL: the operator (row list, row pointers, entries) is immutable, so its loads may overlap the
    // tail of the previous launch; every VECTOR access below comes after pdl_wait().  On the small,
    // latency-bound levels this hides two of the three dependent round trips of a wave.
    pdl_launch_dependents();

    // inactive groups still take part in the shuffles / block reduction below
    int row = 0, start = 0, end = 0;
    if (active) {
        row = INDEXED ? a.rows[k] : a.row0 + (int)k;
        start = a.Ap[row];
        end = a.Ap[row + 1];
    }
    double sum = 0.0, diag = 0.0;
    int jd = -1;
    // chunks of U independent (col,val) loads, then U independent gathers: the per-row latency chain is
    // row-pointer -> entries -> gathers, whatever the row length
    constexpr int U = 4;
    for (int j0 = start + lane; j0 < end; j0 += G * U) {
        int c[U];
        double v[U], xv[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int jj = j0 + u * G;
            const bool ok = jj < end;
            c[u] = ok ? ld_stream_i32(a.Aj + jj) : -1;
            v[u] = ok ? ld_stream_f64(a.Ax + jj) : 0.0;
        }
        pdl_wait();
#pragma unroll
        for (int u = 0; u < U; u++) {
            const bool skip = c[u] < 0 || (kNeedDiag && c[u] == row);
            xv[u] = skip ? 0.0 : ((OP == OP_GS) ? a.x[c[u]] : __ldg(a.x + c[u]));
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (kNeedDiag && c[u] == row && c[u] >= 0) { diag = v[u]; jd = j0 + u * G; }   // later duplicates overwrite
            else sum += v[u] * xv[u];
        }
    }
    pdl_wait();          // rows without entries never entered the loop
    sum = group_sum<G>(sum);
    if (kNeedDiag) {
        // last stored diagonal duplicate wins (relaxation.h:66-69): keep the one with max jj
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) {
            const int jo = __shfl_xor_sync(0xffffffffu, jd, o, G);
            const double dv = __shfl_xor_sync(0xffffffffu, diag, o, G);
            if (jo > jd) { jd = jo; diag = dv; }
        }
    }
    if (active && lane == 0) {
        if (OP == OP_SPMV) {
            a.y[row] = sum;
        } else if (OP == OP_RESID) {
            const double r = a.b[row] - sum;
            a.y[row] = r;
            r2 = r * r;
        } else if (OP == OP_PADD) {
            a.y[row] += sum;
        } else if (OP == OP_JACOBI) {
            const double xi = a.x[row];
            const double bi = a.b[row];
            double xn = xi;
            if (diag != 0.0) xn = (1.0 - a.omega) * xi + a.omega * ((bi - sum) / diag);
            a.y[row] = xn;
            if (a.r != nullptr) {
                const double r = bi - sum - diag * xi;   // residual of the INPUT iterate
                a.r[row] = r;
                r2 = r * r;
            }
        } else {  // OP_GS (omega != 1: sor_gauss_seidel, relaxation.h:116-145)
            if (diag != 0.0) {
                const double g = (a.b[row] - sum) / diag;
                a.y[row] = (a.omega == 1.0) ? g : a.omega * g + (1.0 - a.omega) * a.y[row];
            }
        }
    }
    if ((OP == OP_RESID || OP == OP_JACOBI) && a.partials != nullptr) {
        const double t = block_sum<kCsrThreads>(r2);
        if (threadIdx.x == 0) a.partials[blockIdx.x] = t;
    }
}

// ---------------------------------------------------------------------------------------------
// small vector kernels
// ---------------------------------------------------------------------------------------------
__global__ void fill_kernel(double *x, long long n, double v)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) x[i] = v;
}

// partials[b] = sum of x_i^2 over block b's grid-stride share (fixed grid -> deterministic)
constexpr int kSumsqBlocks = 148 * 8;
__global__ void __launch_bounds__(256) sumsq_partials_kernel(const double *__restrict__ x, long long n,
                                                             double *__restrict__ partials)
{
    double t = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        t += x[i] * x[i];
    t = block_sum<256>(t);
    if (threadIdx.x == 0) partials[blockIdx.x] = t;
}

// partials[b] = sum of x_i*y_i over block b's grid-stride share (fixed grid -> deterministic dot products)
__global__ void __launch_bounds__(256) dot_partials_kernel(const double *__restrict__ x, const double *__restrict__ y,
                                                           long long n, double *__restrict__ partials)
{
    double t = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        t += x[i] * y[i];
    t = block_sum<256>(t);
    if (threadIdx.x == 0) partials[blockIdx.x] = t;
}

// y = a*x + b*y  (Krylov vector updates)
__global__ void axpby_kernel(double a, const double *__restrict__ x, double b, double *__restrict__ y, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) y[i] = a * x[i] + b * y[i];
}

// y = a*x  (first Horner term of the polynomial smoother; never reads y, which may be uninitialised)
__global__ void scale_kernel(double a, const double *__restrict__ x, double *__restrict__ y, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) y[i] = a * x[i];
}

// y += sign * (num / den) * x with the two scalars read from device memory (AMLI step sizes: no host round trip,
// so the cycle stays capturable in a CUDA graph)
__global__ void axpy_ratio_kernel(double *__restrict__ y, const double *__restrict__ x, const double *num,
                                  const double *den, double sign, long long n)
{
    const double a = sign * (num[0] / den[0]);
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) y[i] += a * x[i];
}

// ---------------------------------------------------------------------------------------------
// Householder GMRES / flexible GMRES vector kernels (amgb_solve_gmres; pyamg/krylov/_gmres_householder.py,
// _fgmres.py).  Vectors are in the ORIGINAL numbering: the reflectors single out leading entries.
// ---------------------------------------------------------------------------------------------
// v = (I - 2 w w^T) e_k = (-2 w_k) w + e_k                       (_gmres_householder.py:214-215)
__global__ void hh_unit_reflect_kernel(double *__restrict__ v, const double *__restrict__ w, long long k, long long n)
{
    const double f = -2.0 * w[k];
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        double t = f * w[i];
        if (i == k) t = t + 1.0;
        v[i] = t;
    }
}
// w = [0 ... 0, v_k1 + alpha, v_{k1+1}, ..., v_{n-1}]               (:242-246; k1 = 0: :189-191).  w may alias v.
__global__ void hh_make_w_kernel(double *w, const double *v, long long k1, double alpha, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        double t = (i < k1) ? 0.0 : v[i];
        if (i == k1) t += alpha;
        w[i] = t;
    }
}
__global__ void div_kernel(double *__restrict__ y, double d, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) y[i] = y[i] / d;
}
__global__ void add_at_kernel(double *x, long long i, double v) { x[i] += v; }
// partials[b] = sum of x_i^2 over i >= start of block b's grid-stride share   (norm of v[inner+1:], :239-240)
__global__ void __launch_bounds__(256) sumsq_from_partials_kernel(const double *__restrict__ x, long long start,
                                                                  long long n, double *__restrict__ partials)
{
    double t = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        if (i >= start) t += x[i] * x[i];
    t = block_sum<256>(t);
    if (threadIdx.x == 0) partials[blockIdx.x] = t;
}
// stagnation test (:342-347): partials[b] = max |u_i / x_i| over x_i != 0 (-1 if the share has none)
__global__ void __launch_bounds__(256) maxratio_partials_kernel(const double *__restrict__ u, const double *__restrict__ x,
                                                                long long n, double *__restrict__ partials)
{
    __shared__ double s_max[8];
    double t = -1.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        if (x[i] != 0.0) t = fmax(t, fabs(u[i] / x[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = fmax(t, __shfl_xor_sync(0xffffffffu, t, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < 8; i++) t = fmax(t, s_max[i]);
        partials[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(1024) reduce_max_kernel(const double *partials, int m, double *out)
{
    __shared__ double s_max[32];
    double t = -1.0;
    for (int i = threadIdx.x; i < m; i += 1024) t = fmax(t, partials[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = fmax(t, __shfl_xor_sync(0xffffffffu, t, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < 32; i++) t = fmax(t, s_max[i]);
        *out = t;
    }
}

// ---------------------------------------------------------------------------------------------
// Modified Gram-Schmidt GMRES vector kernels (amgb_solve_gmres with AMGB_FLAG_MGS; pyamg/krylov/_gmres_mgs.py).
// Vectors are in the level-0 numbering: MGS needs only inner products, axpys, A and M.
// ---------------------------------------------------------------------------------------------
// One fused MGS step on v, a grid-stride pass with dot_partials_kernel's grid and order:
//   vprev != nullptr: v -= c * vprev, c = *coef (the previous projection's coefficient, written on the device by the
//                     previous step's reduction)                                          (:253, axpy(vk, v, n, -alpha))
//   dots != nullptr:  dots[b] = block b's partial of <vk, v> with the updated v            (:251, the next coefficient)
//   sq != nullptr:    sq[b]   = block b's partial of <v, v> with the updated v             (:246 normv_old, :256 normv)
// Contraction: nvcc contracts `x - c * p` to one DFMA, fma(-c, p, x), and the sums `t += a * b` to fma(a, b, t) as in
// dot_partials_kernel / sumsq_partials_kernel; many_mgs_step_kernel writes the same expressions per column.
__global__ void __launch_bounds__(256) mgs_step_kernel(double *__restrict__ v, const double *__restrict__ vprev,
                                                       const double *__restrict__ coef, const double *__restrict__ vk,
                                                       long long n, double *__restrict__ dots, double *__restrict__ sq)
{
    const double c = vprev != nullptr ? coef[0] : 0.0;
    double td = 0.0, ts = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        double x = v[i];
        if (vprev != nullptr) {
            x = x - c * vprev[i];
            v[i] = x;
        }
        if (dots != nullptr) td += vk[i] * x;
        if (sq != nullptr) ts += x * x;
    }
    if (dots != nullptr) {
        td = block_sum<256>(td);
        if (threadIdx.x == 0) dots[blockIdx.x] = td;
    }
    if (sq != nullptr) {
        __syncthreads();                           // block_sum's shared partials are reused
        ts = block_sum<256>(ts);
        if (threadIdx.x == 0) sq[blockIdx.x] = ts;
    }
}
// y = x * (1.0 / h) with h = sqrt(*nsq) when h != 0, else y = x (:268-269: scal(1.0/normv, v), a multiply by the
// reciprocal).  The build has no fast-math, so sqrt and the division are IEEE and equal the host's.
__global__ void mgs_scale_kernel(double *__restrict__ y, const double *__restrict__ x, const double *nsq, long long n)
{
    const double h = sqrt(nsq[0]);
    const double r = 1.0 / h;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) y[i] = h != 0.0 ? x[i] * r : x[i];
}

// ---------------------------------------------------------------------------------------------
// Kaczmarz-type sweeps (gauss_seidel_ne / gauss_seidel_nr, relaxation.h:633-657, :684-713): G lanes per row of M
// (= A for NE, = A^T for NR); the rows of one launch share no column (conflict waves), so the scatter updates of
// different rows never touch the same entry of v.
//   NE: delta = (b_i - sum_j m_ij v_j) * Dinv_i * omega ;  v_j += m_ij * delta            (v = x)
//   NR: delta = (sum_j m_ij v_j) * (Dinv_i * omega)     ;  x_i += delta ; v_j -= delta * m_ij   (v = r)
// ---------------------------------------------------------------------------------------------
template <int G, bool NR>
__global__ void __launch_bounds__(kCsrThreads) kaczmarz_kernel(int nrows, const int *__restrict__ rows,
                                                               const int *__restrict__ Mp, const int *__restrict__ Mj,
                                                               const double *__restrict__ Mx, double *v,
                                                               const double *__restrict__ b,
                                                               const double *__restrict__ Dinv, double omega, double *xout)
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
    double sum = 0.0;
    for (int jj = start + lane; jj < end; jj += G) sum += Mx[jj] * v[Mj[jj]];
    sum = group_sum<G>(sum);                       // every lane of the group holds the row's inner product
    if (!active) return;                           // (after the shuffles: inactive groups took part in them)
    double delta;
    if (NR) {
        delta = sum * (Dinv[row] * omega);
        if (lane == 0) xout[row] += delta;
        for (int jj = start + lane; jj < end; jj += G) v[Mj[jj]] -= delta * Mx[jj];
    } else {
        delta = (b[row] - sum) * Dinv[row] * omega;
        for (int jj = start + lane; jj < end; jj += G) v[Mj[jj]] += Mx[jj] * delta;
    }
}

// ---------------------------------------------------------------------------------------------
// multiplicative overlapping Schwarz (relaxation.h:818-880): one warp per subdomain of the launch (subdomains of a
// wave neither read nor write each other's entries).  Every lane forms whole local rows sequentially -- rsum_q =
// (-sum a x) + b, then (T rsum)_q with T the block's stored (pseudo-)inverse -- in the reference's own order, so the
// arithmetic is the sequential code's, bit for bit; all reads of x precede the updates (two warp barriers).
// Shared memory: 2 * max_m doubles per warp.
// ---------------------------------------------------------------------------------------------
constexpr int kSchwarzWarps = 4;
__global__ void __launch_bounds__(kSchwarzWarps * 32) schwarz_kernel(int ndom, const int *__restrict__ doms,
                                                                    const int *__restrict__ Sp, const int *__restrict__ Sj,
                                                                    const long long *__restrict__ Tp,
                                                                    const double *__restrict__ Tx,
                                                                    const int *__restrict__ Ap, const int *__restrict__ Aj,
                                                                    const double *__restrict__ Ax, double *x,
                                                                    const double *__restrict__ b, int max_m)
{
    extern __shared__ __align__(16) unsigned char schwarz_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double *rsum = reinterpret_cast<double *>(schwarz_smem) + (size_t)warp * 2 * max_m;
    double *upd = rsum + max_m;
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
        double r = 0.0;
        for (int jj = Ap[row]; jj < Ap[row + 1]; jj++) r -= Ax[jj] * x[Aj[jj]];
        rsum[q] = r + b[row];
    }
    __syncwarp();
    for (int q = lane; q < m; q += 32) {
        double u = 0.0;
        const double *Trow = Tx + t0 + (long long)q * m;
        for (int c = 0; c < m; c++) u += Trow[c] * rsum[c];
        upd[q] = u;
    }
    __syncwarp();
    for (int q = lane; q < m; q += 32) x[Sj[s0 + q]] += upd[q];
}

// Arnoldi pieces (amgb_arnoldi_run): everything between two host reads stays on the device
__global__ void sqrt_scalar_kernel(double *p) { *p = sqrt(*p); }
// y = x / *den   (next Krylov basis vector: w / ||w|| with the norm in a device scalar)
__global__ void div_dev_kernel(double *__restrict__ y, const double *__restrict__ x, const double *den, long long n)
{
    const double d = den[0];
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) y[i] = x[i] / d;
}
// y *= s (elementwise): the operator diag(s) A of rho(D^-1 A) without forming the scaled matrix
__global__ void mul_kernel(double *__restrict__ y, const double *__restrict__ s, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) y[i] = y[i] * s[i];
}

// out[slot] = sum(partials[0..m)) in a fixed order (single block) -> deterministic norms
__global__ void __launch_bounds__(1024) reduce_partials_kernel(const double *partials, int m,
                                                               double *out)
{
    double t = 0.0;
    for (int i = threadIdx.x; i < m; i += 1024) t += partials[i];
    t = block_sum<1024>(t);
    if (threadIdx.x == 0) *out = t;
}

// y (m) = M (m x n, row-major) * x (n): the cached dense pseudo-inverse of the coarsest
// operator applied to the coarse rhs (pyamg/multilevel.py:717-721, `np.dot(self.P, b)`).
// One warp per row; coarsest grids have 2..500 unknowns, so this is latency-, not bandwidth-bound.
__global__ void dense_matvec_kernel(int m, int n, const double *__restrict__ M,
                                    const double *__restrict__ x, double *__restrict__ y)
{
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int l = threadIdx.x & 31;
    if (w >= m) return;
    double s = 0.0;
    for (int j = l; j < n; j += 32) s += M[(size_t)w * n + j] * x[j];
    s = group_sum<32>(s);
    if (l == 0) y[w] = s;
}

// gather/scatter used for permuted layouts and halo packing: out[i] = in[idx[i]]
__global__ void gather_kernel(const double *__restrict__ in, const int *__restrict__ idx,
                              double *__restrict__ out, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = in[idx[i]];
}

}  // namespace amgb
