// tile_flat_kernel.cuh -- flat-gather tile kernel: by default (AMGB_TILE_FLAT=2) the restrictions of every level and
// the prolongations from level 1 down; AMGB_TILE_FLAT=1 uses it for every tiled operator, 0 never.
//
// Same TMA-staged tiles, same persistent grid and the same five epilogues as csr_tile_kernel (tile_kernels.cuh),
// but the work inside a tile is split the "CSR-stream" way instead of G lanes per row:
//   phase 1  the warp walks the tile's stored entries FLAT (entry e -> lane e mod 32): every lane gathers
//            x[col[e]] for its <= T/32 entries -- all loads independent, every lane busy whatever the row
//            lengths -- and overwrites val[e] with the product in shared memory;
//   phase 2  32/g rows at a time, g lanes add up a row's products out of shared memory (g chosen per tile from
//            its row count) and run the fused epilogue.
// Why: on the coarse operators of the 256^3 hierarchy (19-130 entries per row, 2-11 rows per tile) the
// lanes-per-row walk keeps only ~45 % of the lanes busy (ncu: 14.5 of 32 threads per gather request on level 1)
// and needs two or more dependent gather rounds per tile; here it is one round at full width.
//
// Diagonal (Jacobi / Gauss-Seidel): an entry can only be its row's diagonal if its column lies in the tile's own
// row range; such a candidate (column c) is the diagonal exactly when the entry is stored in row c, i.e. its
// global index lies in [Ap[c], Ap[c+1]) of the staged row pointers; the value then goes to a per-row slot and
// the product is dropped.  Matrices with a diagonal stored twice keep the lanes-per-row kernel (the reference
// lets the last duplicate win; engine.cu checks at upload).
//
// CODED (value codes, see tile_kernels.cuh): the stage holds the entries' 1-byte codes; phase 1 decodes them and
// writes the products to a separate fp64 scratch array, which phase 2 reads.
#pragma once
#include "tile_kernels.cuh"

namespace amgb {

// the stage layout of tile_kernels.cuh this kernel uses: fp64 values or 1-byte value codes (never pair codes: its
// operators, R and the coarse P, are rectangular, so column - row is not a stencil offset)
template <bool CODED>
constexpr int kFlatCode = CODED ? CODE_VAL8 : CODE_NONE;

// phase 1's products: in the stage's own values (fp64), or in a scratch array beside the codes
template <class C, bool CODED>
struct TileFlatProducts {};
template <class C>
struct TileFlatProducts<C, true> {
    double prod[C::T + 16];
};
template <class C, int OP, bool CODED = false>
struct __align__(16) TileFlatWarpSmemT : TileFlatProducts<C, CODED> {
    TileStageT<C, OP, kFlatCode<CODED>> st;          // single stage (TileCfg6 geometry)
    double dslot[(OP == OP_JACOBI || OP == OP_GS) ? C::RMAX : 2];   // diagonal value per row of the tile
    unsigned long long bar;
    unsigned long long pad_;
};
template <class C, int OP, bool CODED = false>
constexpr size_t tile_flat_smem_bytes()
{
    return sizeof(TileFlatWarpSmemT<C, OP, CODED>) * C::WARPS + tile_table_bytes<kFlatCode<CODED>>();
}

__device__ __forceinline__ void fence_proxy_async_smem()
{
#ifndef AMGB_EMU
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}

// launch bounds: 6 CTAs of 8 warps per SM (the residency the tile kernels were tuned to) caps registers at 40
template <int OP, class C, bool PDL, bool CODED = false>
__global__ void __launch_bounds__(C::WARPS * 32, 6) csr_tile_flat_kernel(const TileArgs a)
{
    static_assert(C::STAGES == 1, "flat tile kernel: single-stage geometry only");
    static_assert(C::T % 32 == 0, "flat tile kernel: T must be a multiple of the warp size");
    if (PDL) pdl_launch_dependents();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr bool kNeedDiag = (OP == OP_JACOBI || OP == OP_GS);
    constexpr int EPL = C::T / 32;                    // entries per lane in phase 1
    constexpr int kAl = TileStageVals<C, kFlatCode<CODED>>::kAlign;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    using WS = TileFlatWarpSmemT<C, OP, CODED>;
    WS &ws = reinterpret_cast<WS *>(smem_raw)[warp];
    TileStageT<C, OP, kFlatCode<CODED>> &st = ws.st;
    const void *sdict = load_dict<kFlatCode<CODED>>(a, smem_raw + sizeof(WS) * C::WARPS);
    double *prod;
    if constexpr (CODED) prod = ws.prod;
    else prod = st.val;

    if (lane == 0) {
        mbar_init(&ws.bar, 1);
        fence_mbar_init();
    }
    if (CODED) __syncthreads();   // the table is complete
    else __syncwarp();
    const unsigned long long pol_first = policy_evict_first();
    const unsigned long long pol_last = policy_evict_last();

    const int nwarps = gridDim.x * C::WARPS;
    int t = a.tile_begin + blockIdx.x * C::WARPS + warp;
    unsigned phase = 0;
    double r2 = 0.0;

    bool requested = false;
    if (PDL) {
        if (lane == 0 && t < a.tile_end) tile_issue<C, OP, kFlatCode<CODED>, 1>(a, t, st, &ws.bar, pol_first);
        pdl_wait();
        if (lane == 0 && t < a.tile_end) tile_issue<C, OP, kFlatCode<CODED>, 2>(a, t, st, &ws.bar, pol_first);
        requested = true;
    }
    for (; t < a.tile_end; t += nwarps) {
        if (lane == 0 && !requested) tile_issue<C, OP, kFlatCode<CODED>>(a, t, st, &ws.bar, pol_first);
        requested = false;

        const TileDesc d0 = a.tiles[t], d1 = a.tiles[t + 1];
        const int row0 = d0.row0, nrows = d1.row0 - d0.row0;
        const int s0 = d0.nz0, len = d1.nz0 - d0.nz0;
        if (kNeedDiag && len <= C::T) {
            // reset the diagonal slots while the copy is in flight (the TMA never writes them)
            for (int lr = lane; lr < nrows; lr += 32) ws.dslot[lr] = 0.0;
        }
        mbar_wait(&ws.bar, phase);
        phase ^= 1u;

        if (len <= C::T) {
            const int soff = s0 & ~(kAl - 1);         // smem index = global entry index - soff
            const int poff = row0 & ~3;
            const int voff = row0 & ~1;
            const int e0 = s0 - soff;                 // first / one-past-last staged entry of the tile
            const int e1 = e0 + len;
            if (kNeedDiag) __syncwarp();              // slots are zero before any lane stores a diagonal
            // ---- phase 1: flat gather, products in place ------------------------------------------
            {
                int c[EPL];
                double xv[EPL];
#pragma unroll
                for (int u = 0; u < EPL; u++) {
                    const int e = e0 + lane + 32 * u;
                    c[u] = (e < e1) ? st.col[e] : -1;
                }
#pragma unroll
                for (int u = 0; u < EPL; u++) {
                    if (c[u] >= 0) {
                        if (a.hints) xv[u] = (OP == OP_GS) ? ld_x_hint(a.x + c[u], pol_last) : ld_x_hint_nc(a.x + c[u], pol_last);
                        else xv[u] = (OP == OP_GS) ? a.x[c[u]] : __ldg(a.x + c[u]);
                    } else {
                        xv[u] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < EPL; u++) {
                    const int e = e0 + lane + 32 * u;
                    if (c[u] < 0) continue;
                    const double v = stage_val<kFlatCode<CODED>>(st, e, sdict);   // read here, not held across the gathers: registers = residency
                    double p = v * xv[u];
                    if (kNeedDiag && c[u] >= row0 && c[u] < row0 + nrows) {
                        // candidate: is entry e stored in row c[u]?  (row r holds global entries Ap[r] .. Ap[r+1]-1)
                        const int ge = e + soff;
                        const int lr = c[u] - row0;
                        if (ge >= st.ptr[row0 + lr - poff] && ge < st.ptr[row0 + lr + 1 - poff]) {
                            ws.dslot[lr] = v;
                            p = 0.0;                   // the reference skips the diagonal term
                        }
                    }
                    prod[e] = p;
                }
            }
            __syncwarp();
            // ---- phase 2: g lanes per row add the products up, fused epilogue -------------------------
            int g = 32;                               // largest power of two with g * nrows <= 32 (at least 1)
            while (g > 1 && g * nrows > 32) g >>= 1;
            const int rpp = 32 / g;
            const int sub = lane & (g - 1), grp = lane / g;
            for (int rbase = 0; rbase < nrows; rbase += rpp) {
                const int lr = rbase + grp;
                const bool active = lr < nrows;
                const int row = row0 + lr;
                int jb = 0, je = 0;
                if (active) {
                    jb = st.ptr[row - poff] - soff;
                    je = st.ptr[row - poff + 1] - soff;
                }
                double sum = 0.0;
                for (int jj = jb + sub; jj < je; jj += g) sum += prod[jj];
                for (int o = g >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                if (active && sub == 0) {
                    if (OP == OP_SPMV) {
                        a.y[row] = sum;
                    } else if (OP == OP_RESID) {
                        const double r = st.bseg[row - voff] - sum;
                        a.y[row] = r;
                        r2 += r * r;
                    } else if (OP == OP_PADD) {
                        a.y[row] += sum;
                    } else if (OP == OP_JACOBI) {
                        const double xi = st.xseg[row - voff], bi = st.bseg[row - voff];
                        const double diag = ws.dslot[lr];
                        double xn = xi;
                        if (diag != 0.0) xn = (1.0 - a.omega) * xi + a.omega * ((bi - sum) / diag);
                        a.y[row] = xn;
                        if (a.r != nullptr) {
                            const double r = bi - sum - diag * xi;
                            a.r[row] = r;
                            r2 += r * r;
                        }
                    } else {
                        const double diag = ws.dslot[lr];
                        if (diag != 0.0) {
                            const double gs = (st.bseg[row - voff] - sum) / diag;
                            a.y[row] = (a.omega == 1.0) ? gs : a.omega * gs + (1.0 - a.omega) * a.y[row];
                        }
                    }
                }
            }
        } else {
            // a single row longer than a tile: the whole warp strides over it in global memory
            const int row = row0;
            double sum = 0.0, diag = 0.0;
            int jd = -1;
            for (int jj = s0 + lane; jj < s0 + len; jj += 32) {
                const int c = ld_stream_i32(a.Aj + jj);
                const double v = global_val<kFlatCode<CODED>>(a, jj, sdict);
                const double xv = (OP == OP_GS) ? a.x[c] : __ldg(a.x + c);
                if (kNeedDiag && c == row) { diag = v; jd = jj; }
                else sum += v * xv;
            }
            sum = group_sum<32>(sum);
            if (kNeedDiag) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const int jo = __shfl_xor_sync(0xffffffffu, jd, o);
                    const double dv = __shfl_xor_sync(0xffffffffu, diag, o);
                    if (jo > jd) { jd = jo; diag = dv; }
                }
            }
            if (lane == 0) {
                if (OP == OP_SPMV) a.y[row] = sum;
                else if (OP == OP_RESID) { const double r = a.b[row] - sum; a.y[row] = r; r2 += r * r; }
                else if (OP == OP_PADD) a.y[row] += sum;
                else if (OP == OP_JACOBI) {
                    const double xi = a.x[row], bi = a.b[row];
                    a.y[row] = (diag != 0.0) ? (1.0 - a.omega) * xi + a.omega * ((bi - sum) / diag) : xi;
                    if (a.r != nullptr) { const double r = bi - sum - diag * xi; a.r[row] = r; r2 += r * r; }
                } else if (diag != 0.0) {
                    const double gs = (a.b[row] - sum) / diag;
                    a.y[row] = (a.omega == 1.0) ? gs : a.omega * gs + (1.0 - a.omega) * a.y[row];
                }
            }
        }
        // the products were written through the generic proxy; the next tile arrives through the async proxy
        fence_proxy_async_smem();
        __syncwarp();             // every lane is done with this stage before the TMA refills it
    }
    if ((OP == OP_RESID || OP == OP_JACOBI) && a.partials != nullptr) {
        const double tsum = block_sum<C::WARPS * 32>(r2);
        if (threadIdx.x == 0) a.partials[blockIdx.x] = tsum;
    }
}

}  // namespace amgb
