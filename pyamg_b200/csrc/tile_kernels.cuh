// tile_kernels.cuh -- the sm_90a streaming kernel of the V-cycle: CSR row segments staged in shared
// memory by the TMA (1-D bulk copies, cp.async.bulk -> SASS UBLKCP) with mbarrier completion.
//
// Why: the hot path is HBM-bound CSR traffic (12 B per stored entry, 0.17 flop/B).  A lanes-per-row
// kernel (csr_kernels.cuh) keeps only a few hundred bytes per warp in flight and pays a dependent
// row-pointer -> entries -> gather latency chain per row group.  Here every warp owns a ring of
// shared-memory stages; one elected lane asks the TMA for the NEXT tile's contiguous segments
// (values, column indices, row pointers, and the b / x_old slices the epilogue needs -- each a single
// 16-B-aligned bulk copy) while the warp reduces the CURRENT tile out of shared memory.  The copy
// engine, not the LSU, streams the operator; the warps only issue the x gathers and the fused
// epilogue store.  Bytes in flight per SM = warps x stage size, independent of register pressure.
//
// Tiles are built on the host at upload (engine.cu build_tiles): whole rows, at most T stored entries
// and RMAX rows, never crossing a Gauss-Seidel wave boundary; a row longer than T is a tile of its own
// and is streamed straight from global memory.  Work distribution is static (tile t -> warp t mod
// #warps), the grid persistent: all SMs x resident CTAs.
//
// L2 policy: the operator stream is read exactly once per launch -> evict-first; the gathered vector
// is re-read by every row that references it (and, for multi-colour Gauss-Seidel, by every wave) ->
// evict-last, so it survives in the 50 MB L2 of the H100 while the operator streams past it.
//
// Epilogues (template OP, same semantics as csr_kernels.cuh / the reference, file:line there):
//   OP_SPMV, OP_RESID (+|r|^2), OP_PADD, OP_JACOBI (+ optional residual by-product), OP_GS (rows of one
//   wave, contiguous thanks to the wave-major row permutation applied at upload; + optional residual of those rows
//   when the wave is the last one of a sweep; entries with column -1 are the padding of a zero-start copy, engine.cu
//   build_zero_start, and add no term).
//
// Value codes (CODE_VAL8): an operator with at most 256 distinct values (by bit pattern) is also stored as one
// byte per entry indexing a table of those doubles (engine.cu upload_csr).  The coded variants stream the codes in
// place of the 8-byte values (5 B per entry instead of 12) and decode from a copy of the table in shared memory.
// The decoded double is the stored double and nothing else changes, so the results are bit-identical.
//
// Pair codes (CODE_PAIR8): an operator whose entries take at most 256 distinct (value bit pattern, column - row)
// pairs -- a constant-coefficient stencil in a fixed row order, such as level 0 of a 7-point Poisson hierarchy in
// red-black wave-major order (15 pairs) -- stores one byte per entry indexing a table of (value, column - row).
// These launches stream neither values nor columns: 1 B per entry.  The column is rebuilt as row + delta, which is
// the stored column, so the results are again bit-identical.
//
// Row codes (csr_rowcode_kernel): a pair-coded operator on one lane per row whose rows take at most 256 distinct
// sequences of pair codes, none longer than kRowCodeMaxLen -- 56 at level 0 of the 7-point Poisson hierarchy in
// red-black wave-major order, whatever the grid -- stores one byte per row naming its sequence.  Those launches walk
// the same tile list with the same tile -> warp -> lane -> row assignment and grid, but stream no entries and no row
// pointers, so nothing is left for the TMA: every per-lane load (row code, b, old x) is a plain coalesced load, and
// each warp loads the next tile's while it reduces the current one.  Sums, epilogue and partials are those of
// csr_tile_kernel in the same order, so the results are bit-identical.
#pragma once
#include "csr_kernels.cuh"

namespace amgb {

struct TileDesc { int row0; int nz0; };   // tile t = rows [row0[t], row0[t+1]), entries [nz0[t], nz0[t+1])

// how a tile launch reads its entries: fp64 value + column, 1-byte value code + column, or 1-byte pair code
enum : int { CODE_NONE = 0, CODE_VAL8 = 1, CODE_PAIR8 = 2 };

struct __align__(16) PairCode {   // one pair-code table entry: the value and the column offset from the row
    double v;
    int delta;
    int pad_;
};

// Row codes: one table entry per distinct row, the pair codes of its entries in stored order (16 B: one shared-memory
// load per row)
constexpr int kRowCodeMaxLen = 15;
struct __align__(16) RowPattern {
    unsigned char len;
    unsigned char pair[kRowCodeMaxLen];
};

struct TileArgs {
    const TileDesc *tiles;   // n_tiles + 1 descriptors (sentinel last)
    int tile_begin, tile_end;
    const int *Ap;
    const int *Aj;
    const double *Ax;
    // one code per entry (padded to 16-entry groups), or, row-coded (patterns set), one per row; nullptr: fp64 values
    const unsigned char *codes = nullptr;
    union {                                 // (one pointer: the kernels' parameter block keeps its size and layout)
        const double *dict = nullptr;       // value codes: the ndict (<= kMaxCodes) values the codes index
        const RowPattern *patterns;         // row codes: the kMaxCodes row patterns the codes index, entries -> pairs
    };
    const PairCode *pairs = nullptr;        // pair codes (codes index this table instead of dict), or nullptr
    int ndict = 0;
    const double *x;
    const double *b;
    double *y;
    double *r;
    double omega;
    double *partials;        // one per CTA (grid is fixed), or nullptr
    int hints;               // 1: L2 eviction hints (operator stream evict-first, x gathers evict-last)
};

constexpr int kMaxCodes = 256;

// Resident CTAs per SM the tile launches of each epilogue aim for (SpMV, residual, prolong+add, Jacobi, Gauss-Seidel;
// engine.cu tile_cfg_op): the persistent grid is this many CTAs per SM
constexpr int kTileCtas[5] = {6, 7, 6, 5, 6};

// Tile geometry (compile-time): T stored entries and RMAX rows per tile, ring depth, warps per CTA.
// Shared memory per CTA = WARPS * STAGES * (12 T + 20 RMAX + ~150) bytes; what is left of the
// 228 KB/SM is L1 for the x gathers, so smaller tiles trade TMA efficiency for gather hit rate.
template <int T_, int RMAX_, int STAGES_, int WARPS_>
struct TileCfg {
    static constexpr int T = T_, RMAX = RMAX_, STAGES = STAGES_, WARPS = WARPS_;
};
using TileCfg0 = TileCfg<512, 128, 2, 8>;
using TileCfg1 = TileCfg<256, 64, 2, 8>;
using TileCfg4 = TileCfg<256, 64, 1, 8>;     // single stage, ~48 warps/SM: cross-warp overlap only
using TileCfg6 = TileCfg<224, 64, 1, 8>;     // 32 seven-point rows per tile; 7-8 CTAs/SM = 56-64 warps/SM
using TileCfg7 = TileCfg<352, 64, 1, 8>;     // denser coarse operators (~19-36 entries per row): 16 rows of 19 entries
                                             // fill both passes of a G = 2 warp (224 entries hold 11 such rows: 69 % of
                                             // the lanes, ncu profiles/r02_ncu_kernels.csv: 17.5 threads per instruction)

// A stage's entry values: fp64, staged from 4-entry (16-B) boundaries, or 1-byte codes, staged from 16-entry
// boundaries so that the code copy stays 16-B aligned.  kAlign entries, widened on both sides of the tile.
// kCol: the stage also holds the entries' columns (pair codes carry the column in the code).
template <class C, int CODE>
struct TileStageVals {
    static constexpr int kAlign = 4, kE = C::T + 8;
    static constexpr bool kCol = true;
    static constexpr unsigned kVB = 8;     // bytes per entry of the value stream
    double val[kE];
};
template <class C>
struct TileStageVals<C, CODE_VAL8> {
    static constexpr int kAlign = 16, kE = C::T + 32;
    static constexpr bool kCol = true;
    static constexpr unsigned kVB = 1;
    unsigned char code[kE];
};
template <class C>
struct TileStageVals<C, CODE_PAIR8> {
    static constexpr int kAlign = 16, kE = C::T + 32;
    static constexpr bool kCol = false;
    static constexpr unsigned kVB = 1;
    unsigned char code[kE];
};

// the b / x_old slices are staged only for the epilogues that read them: shared memory is what limits
// the number of resident warps, and resident warps are what hides the gather latency
template <class C, int OP, int CODE = CODE_NONE>
struct __align__(16) TileStageT : TileStageVals<C, CODE> {
    static constexpr bool kB = (OP == OP_RESID || OP == OP_JACOBI || OP == OP_GS);
    static constexpr bool kX = (OP == OP_JACOBI);
    double bseg[kB ? C::RMAX + 4 : 2];    // b[row0..row1)
    double xseg[kX ? C::RMAX + 4 : 2];    // x[row0..row1), old iterate
    int col[TileStageVals<C, CODE>::kCol ? TileStageVals<C, CODE>::kE : 4];
    int ptr[C::RMAX + 8];
};
template <class C, int OP, int CODE = CODE_NONE>
struct __align__(16) TileWarpSmemT {
    TileStageT<C, OP, CODE> st[C::STAGES];
    unsigned long long bar[C::STAGES];
    unsigned long long pad_;
};
// bytes of a coded variant's table, kept behind the warps' stages once per CTA
template <int CODE>
constexpr size_t tile_table_bytes()
{
    return CODE == CODE_VAL8 ? kMaxCodes * sizeof(double) : CODE == CODE_PAIR8 ? kMaxCodes * sizeof(PairCode) : 0;
}
template <class C, int OP, int CODE = CODE_NONE>
constexpr size_t tile_smem_bytes() { return sizeof(TileWarpSmemT<C, OP, CODE>) * C::WARPS + tile_table_bytes<CODE>(); }

// Resident CTAs per SM of the launches of geometry C and epilogue OP on an H100 (228 KB of shared memory per SM), as
// engine.cu tile_cfg_ctas sizes the persistent grid (from the fp64 stage, whose grid the coded launches keep, capped by
// kTileCtas).  csr_tile_kernel is compiled to fit this many CTAs in the register file, so the whole grid is resident.
template <class C, int OP>
constexpr int tile_ctas_per_sm()
{
    const int by_smem = (int)(233472 / (tile_smem_bytes<C, OP>() + 1024));
    const int by_threads = 2048 / (C::WARPS * 32);
    const int c = by_smem < by_threads ? by_smem : by_threads;
    return c < 1 ? 1 : (c < kTileCtas[OP] ? c : kTileCtas[OP]);
}

// Value of staged entry jj: the fp64 value, or the value or pair code's entry in the CTA's table
template <int CODE, class S>
__device__ __forceinline__ double stage_val(const S &st, int jj, const void *table)
{
    if constexpr (CODE == CODE_VAL8) return static_cast<const double *>(table)[st.code[jj]];
    else if constexpr (CODE == CODE_PAIR8) return static_cast<const PairCode *>(table)[st.code[jj]].v;
    else return st.val[jj];
}

// Column of staged entry jj of row `row`
template <int CODE, class S>
__device__ __forceinline__ int stage_col(const S &st, int jj, int row, const void *table)
{
    if constexpr (CODE == CODE_PAIR8) return row + static_cast<const PairCode *>(table)[st.code[jj]].delta;
    else return st.col[jj];
}

__device__ __forceinline__ unsigned ld_stream_u8(const unsigned char *p)
{
#ifdef AMGB_EMU
    return *p;
#else
    unsigned v;
    asm volatile("ld.global.nc.L1::no_allocate.u8 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
#endif
}

// Value of entry jj of a row streamed from global memory (a row longer than a tile)
template <int CODE>
__device__ __forceinline__ double global_val(const TileArgs &a, int jj, const void *table)
{
    if constexpr (CODE == CODE_VAL8) return static_cast<const double *>(table)[ld_stream_u8(a.codes + jj)];
    else return ld_stream_f64(a.Ax + jj);
}

// Column and value of entry jj of row `row`, streamed from global memory (a row longer than a tile)
template <int CODE>
__device__ __forceinline__ void global_entry(const TileArgs &a, int jj, int row, const void *table, int &c, double &v)
{
    if constexpr (CODE == CODE_PAIR8) {
        const PairCode p = static_cast<const PairCode *>(table)[ld_stream_u8(a.codes + jj)];
        c = row + p.delta;
        v = p.v;
    } else {
        c = ld_stream_i32(a.Aj + jj);
        v = global_val<CODE>(a, jj, table);
    }
}

// The coded variant's table: copied to shared memory once per CTA by all its threads (it is immutable, so a
// programmatically-launched kernel may do this before waiting for its predecessor).  Returns its address.
template <int CODE>
__device__ __forceinline__ const void *load_dict(const TileArgs &a, unsigned char *table)
{
    if constexpr (CODE == CODE_VAL8) {
        double *d = reinterpret_cast<double *>(table);
        for (int i = threadIdx.x; i < a.ndict; i += blockDim.x) d[i] = __ldg(a.dict + i);
        return d;
    } else if constexpr (CODE == CODE_PAIR8) {
        PairCode *d = reinterpret_cast<PairCode *>(table);
        for (int i = threadIdx.x; i < a.ndict; i += blockDim.x) d[i] = a.pairs[i];
        return d;
    } else {
        return nullptr;
    }
}

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count)
{
#ifdef AMGB_EMU
    ::emu::mbar_init(bar, count);
#else
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
#endif
}
__device__ __forceinline__ void fence_mbar_init()
{
#ifndef AMGB_EMU
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes)
{
#ifdef AMGB_EMU
    ::emu::mbar_arrive_expect_tx(bar, bytes);
#else
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
#endif
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity)
{
#ifdef AMGB_EMU
    ::emu::mbar_wait(bar, parity);
#else
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
#endif
}
__device__ __forceinline__ unsigned long long policy_evict_first()
{
#ifdef AMGB_EMU
    return 0ull;
#else
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
#endif
}
__device__ __forceinline__ unsigned long long policy_evict_last()
{
#ifdef AMGB_EMU
    return 0ull;
#else
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
#endif
}
// 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier (TMA, SASS UBLKCP)
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar)
{
#ifdef AMGB_EMU
    ::emu::bulk_g2s(dst, src, bytes, bar);
#else
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
#endif
}
__device__ __forceinline__ void bulk_g2s_hint(void *dst, const void *src, unsigned bytes, unsigned long long *bar,
                                              unsigned long long policy)
{
#ifdef AMGB_EMU
    (void)policy;
    ::emu::bulk_g2s(dst, src, bytes, bar);
#else
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
#endif
}
__device__ __forceinline__ double ld_x_hint_nc(const double *p, unsigned long long policy)
{
#ifdef AMGB_EMU
    (void)policy;
    return *p;
#else
    double v;
    asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(policy));
    return v;
#endif
}
__device__ __forceinline__ double ld_x_hint(const double *p, unsigned long long policy)
{
#ifdef AMGB_EMU
    (void)policy;
    return *p;
#else
    double v;
    asm volatile("ld.global.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(policy) : "memory");
    return v;
#endif
}

// Gathers a lane of csr_tile_kernel issues back to back: its next kTileBatch entries' columns are read from the stage,
// their x loads issued, and only then are the products summed (in stored order), so that a lane waits for one L2
// round trip per batch rather than per entry.  4 keeps the dense-geometry kernels free of spills at the register
// bound of their grid (8 spills 24-32 B).
constexpr int kTileBatch = 4;

// Lane entries j0, j0 + G, ... (kTileBatch of them, those below je) of row `row` in a stage: columns, then the x
// gathers back to back (OP_GS: zero-start padding, c = -1, loads x[0] and adds no term)
template <int G, int OP, int CODE, class S>
__device__ __forceinline__ void stage_gather(const TileArgs &a, const S &st, int j0, int je, int row,
                                             const void *table, unsigned long long pol_last, int (&c)[kTileBatch],
                                             double (&xv)[kTileBatch])
{
#pragma unroll
    for (int k = 0; k < kTileBatch; k++) {
        const int jj = j0 + k * G;
        c[k] = (jj < je) ? stage_col<CODE>(st, jj, row, table) : 0;
    }
#pragma unroll
    for (int k = 0; k < kTileBatch; k++) {
        xv[k] = 0.0;
        if (j0 + k * G < je) {
            const int cx = (OP == OP_GS && c[k] < 0) ? 0 : c[k];
            if (a.hints) xv[k] = (OP == OP_GS) ? ld_x_hint(a.x + cx, pol_last) : ld_x_hint_nc(a.x + cx, pol_last);
            else xv[k] = (OP == OP_GS) ? a.x[cx] : __ldg(a.x + cx);
        }
    }
}

// The per-row epilogue of the tile-list kernels (csr_tile_kernel, csr_rowcode_kernel), one definition so that they
// cannot drift apart: what row `row` writes from its sum of products `sum` (the diagonal left out for Jacobi and
// Gauss-Seidel), its diagonal, b_i and (Jacobi) the old x_i.  b_i and x_i come from accessors, read only where the
// epilogue needs them.  Returns the row's new x for OP_GS, 0 otherwise.
template <int OP, class BI, class XI>
__device__ __forceinline__ double tile_row_epilogue(const TileArgs &a, int row, double sum, double diag, BI b_i,
                                                    XI x_i, double &r2)
{
    double xn = 0.0;
    if (OP == OP_SPMV) {
        a.y[row] = sum;
    } else if (OP == OP_RESID) {
        const double r = b_i() - sum;
        a.y[row] = r;
        r2 += r * r;
    } else if (OP == OP_PADD) {
        a.y[row] += sum;
    } else if (OP == OP_JACOBI) {
        const double xi = x_i(), bi = b_i();
        double xj = xi;
        if (diag != 0.0) xj = (1.0 - a.omega) * xi + a.omega * ((bi - sum) / diag);
        a.y[row] = xj;
        if (a.r != nullptr) {
            const double r = bi - sum - diag * xi;
            a.r[row] = r;
            r2 += r * r;
        }
    } else {
        if (diag != 0.0) {
            const double g = (b_i() - sum) / diag;
            xn = (a.omega == 1.0) ? g : a.omega * g + (1.0 - a.omega) * a.y[row];
            a.y[row] = xn;
        } else if (a.r != nullptr) {
            xn = a.y[row];
        }
    }
    return xn;
}

// The residual a sweep's last Gauss-Seidel wave writes for its row, from rs = (A x)_i with the row's new x
__device__ __forceinline__ void tile_row_residual(const TileArgs &a, int row, double bi, double rs, double &r2)
{
    const double r = bi - rs;
    a.r[row] = r;
    r2 += r * r;
}

// One lane: ask the TMA for tile t's segments.  Every source starts on a 16-byte boundary: entry ranges
// are widened to multiples of 4 entries (16 with 1-byte codes), vector ranges to multiples of 2 (the arrays are
// padded at upload).
// PART: bit 0 = arm the barrier for the whole tile and copy the immutable operator segments, bit 1 = copy the
// vector segments (b / x_old).  The split lets a programmatically-launched kernel (PDL) fetch its first
// operator tile while the previous launch is still writing the vectors.
template <class C, int OP, int CODE, int PART = 3>
__device__ __forceinline__ void tile_issue(const TileArgs &a, int t, TileStageT<C, OP, CODE> &st,
                                           unsigned long long *bar, unsigned long long pol)
{
    const TileDesc d0 = a.tiles[t], d1 = a.tiles[t + 1];
    const int len = d1.nz0 - d0.nz0;
    if (len > C::T) {              // long row: streamed from global memory, nothing to stage
        if (PART & 1) mbar_expect_tx(bar, 0);
        return;
    }
    using V = TileStageVals<C, CODE>;
    constexpr bool kB = (OP == OP_RESID || OP == OP_JACOBI || OP == OP_GS);
    constexpr bool kX = (OP == OP_JACOBI);
    constexpr int kAl = V::kAlign;
    const int s4 = d0.nz0 & ~(kAl - 1);
    const int cnt = ((d1.nz0 + kAl - 1) & ~(kAl - 1)) - s4;
    const int r4 = d0.row0 & ~3;
    const int rcnt = ((d1.row0 + 1 + 3) & ~3) - r4;
    const int v2 = d0.row0 & ~1;
    const int vcnt = ((d1.row0 + 1) & ~1) - v2;
    if (PART & 1) {
        constexpr unsigned kEB = V::kVB + (V::kCol ? 4u : 0u);     // operator bytes per staged entry
        mbar_expect_tx(bar, (unsigned)(cnt * kEB + rcnt * 4 + ((kB ? 1 : 0) + (kX ? 1 : 0)) * vcnt * 8));
        if (cnt > 0) {
            void *vdst;
            const void *vsrc;
            if constexpr (CODE != CODE_NONE) { vdst = st.code; vsrc = a.codes + s4; }
            else { vdst = st.val; vsrc = a.Ax + s4; }
            if (a.hints) {
                bulk_g2s_hint(vdst, vsrc, (unsigned)cnt * V::kVB, bar, pol);
                if (V::kCol) bulk_g2s_hint(st.col, a.Aj + s4, (unsigned)cnt * 4u, bar, pol);
            } else {
                bulk_g2s(vdst, vsrc, (unsigned)cnt * V::kVB, bar);
                if (V::kCol) bulk_g2s(st.col, a.Aj + s4, (unsigned)cnt * 4u, bar);
            }
        }
        bulk_g2s(st.ptr, a.Ap + r4, (unsigned)rcnt * 4u, bar);
    }
    if (PART & 2) {
        if (kB && vcnt > 0) bulk_g2s(st.bseg, a.b + v2, (unsigned)vcnt * 8u, bar);
        if (kX && vcnt > 0) bulk_g2s(st.xseg, a.x + v2, (unsigned)vcnt * 8u, bar);
    }
}

// G lanes per row inside a tile (G = 1: thread per row -- 5/7-point stencils; larger G for the
// denser coarse operators).  32/G rows are reduced per pass.
// PDL = true (opt-in AMGB_TILE_PDL=1, launched with the programmatic-stream-serialization attribute): the
// kernel may start while its predecessor still runs; it arms its barriers and fetches the operator segments
// of its first tile(s), then waits for the predecessor before any vector (x, b, y, r) is touched.
// CODE: CODE_VAL8 streams value codes (TileArgs::codes) and decodes them from the table in shared memory;
// CODE_PAIR8 streams pair codes and decodes value and column from theirs (TileArgs::pairs).
template <int G, int OP, class C, bool PDL = false, int CODE = CODE_NONE>
__global__ void __launch_bounds__(C::WARPS * 32, (tile_ctas_per_sm<C, OP>())) csr_tile_kernel(const TileArgs a)
{
    if (PDL) pdl_launch_dependents();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr bool kNeedDiag = (OP == OP_JACOBI || OP == OP_GS);
    constexpr int RPP = 32 / G;                       // rows per pass
    constexpr int STAGES = C::STAGES;
    constexpr int kAl = TileStageVals<C, CODE>::kAlign;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sub = lane & (G - 1), grp = lane / G;
    using WS = TileWarpSmemT<C, OP, CODE>;
    WS &ws = reinterpret_cast<WS *>(smem_raw)[warp];
    const void *sdict = load_dict<CODE>(a, smem_raw + sizeof(WS) * C::WARPS);

    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; s++) mbar_init(&ws.bar[s], 1);
        fence_mbar_init();
    }
    if (CODE != CODE_NONE) __syncthreads();   // the table is complete
    else __syncwarp();
    const unsigned long long pol_first = policy_evict_first();
    const unsigned long long pol_last = policy_evict_last();

    const int nwarps = gridDim.x * C::WARPS;
    // consecutive tiles go to the warps of one CTA: neighbouring rows share x lines in L1
    int t = a.tile_begin + blockIdx.x * C::WARPS + warp;
    unsigned phase = 0;       // bit s = parity to wait for on stage s
    double r2 = 0.0;

    // tiles whose operator segments are requested before the wait: the ring's prologue, or (single stage) tile t
    constexpr int kPre = (STAGES > 1) ? STAGES - 1 : 1;
    if (PDL) {
        if (lane == 0) {
#pragma unroll
            for (int s = 0; s < kPre; s++)
                if (t + s * nwarps < a.tile_end)
                    tile_issue<C, OP, CODE, 1>(a, t + s * nwarps, ws.st[s], &ws.bar[s], pol_first);
        }
        pdl_wait();               // every thread: the predecessor's vectors are complete and visible from here on
        if (lane == 0) {
#pragma unroll
            for (int s = 0; s < kPre; s++)
                if (t + s * nwarps < a.tile_end)
                    tile_issue<C, OP, CODE, 2>(a, t + s * nwarps, ws.st[s], &ws.bar[s], pol_first);
        }
    } else if (lane == 0) {
#pragma unroll
        for (int s = 0; s < STAGES - 1; s++)
            if (t + s * nwarps < a.tile_end) tile_issue<C, OP, CODE>(a, t + s * nwarps, ws.st[s], &ws.bar[s], pol_first);
    }
    int stage = 0;
    bool requested = PDL && STAGES == 1;      // single stage + PDL: the first tile was requested above
    for (; t < a.tile_end; t += nwarps) {
        // keep the ring full: the stage consumed in the previous iteration is free again
        const int tn = t + (STAGES - 1) * nwarps;
        const int sn = (stage + STAGES - 1) % STAGES;
        if (lane == 0 && tn < a.tile_end && !requested) tile_issue<C, OP, CODE>(a, tn, ws.st[sn], &ws.bar[sn], pol_first);
        requested = false;

        const TileDesc d0 = a.tiles[t], d1 = a.tiles[t + 1];
        const int row0 = d0.row0, nrows = d1.row0 - d0.row0;
        const int s0 = d0.nz0, len = d1.nz0 - d0.nz0;
        mbar_wait(&ws.bar[stage], (phase >> stage) & 1u);
        phase ^= 1u << stage;
        const TileStageT<C, OP, CODE> &st = ws.st[stage];

        if (len <= C::T) {
            const int soff = s0 & ~(kAl - 1);         // smem index = global entry index - soff
            const int poff = row0 & ~3;
            const int voff = row0 & ~1;
            for (int rbase = 0; rbase < nrows; rbase += RPP) {
                const int lr = rbase + grp;
                const bool active = lr < nrows;
                const int row = row0 + lr;
                int jb = 0, je = 0;
                if (active) {
                    jb = st.ptr[row - poff] - soff;
                    je = st.ptr[row - poff + 1] - soff;
                }
                double sum = 0.0, diag = 0.0;
                int jd = -1;
                for (int j0 = jb + sub; j0 < je; j0 += kTileBatch * G) {
                    int c[kTileBatch];
                    double xv[kTileBatch];
                    stage_gather<G, OP, CODE>(a, st, j0, je, row, sdict, pol_last, c, xv);
#pragma unroll
                    for (int k = 0; k < kTileBatch; k++) {
                        const int jj = j0 + k * G;
                        if (jj < je) {
                            const double v = stage_val<CODE>(st, jj, sdict);
                            if (kNeedDiag && c[k] == row) {
                                diag = v;
                                jd = jj;
                            } else if (OP != OP_GS || c[k] >= 0) {    // zero-start padding (c = -1): no term
                                sum += v * xv[k];
                            }
                        }
                    }
                }
                if (G > 1) {
                    sum = group_sum<G>(sum);
                    if (kNeedDiag) {
#pragma unroll
                        for (int o = G / 2; o > 0; o >>= 1) {
                            const int jo = __shfl_xor_sync(0xffffffffu, jd, o, G);
                            const double dv = __shfl_xor_sync(0xffffffffu, diag, o, G);
                            if (jo > jd) { jd = jo; diag = dv; }
                        }
                    }
                }
                double xn = 0.0;      // OP_GS: the row's new value
                if (active && sub == 0) {
                    xn = tile_row_epilogue<OP>(a, row, sum, diag, [&] { return st.bseg[row - voff]; },
                                               [&] { return st.xseg[row - voff]; }, r2);
                }
                if (OP == OP_GS && a.r != nullptr) {
                    // residual of the sweep's LAST wave, from the staged tile: no later wave changes these rows' x
                    // neighbours and rows of one wave never read each other, so r = b - A x is final here.  Summed as
                    // OP_RESID sums it (same lanes, same order), with the new x_i where the row reads itself.
                    if (G > 1) xn = __shfl_sync(0xffffffffu, xn, lane & ~(G - 1));
                    double rs = 0.0;
                    for (int j0 = jb + sub; j0 < je; j0 += kTileBatch * G) {
                        int c[kTileBatch];
                        double xv[kTileBatch];
                        stage_gather<G, OP, CODE>(a, st, j0, je, row, sdict, pol_last, c, xv);
#pragma unroll
                        for (int k = 0; k < kTileBatch; k++)
                            if (j0 + k * G < je)
                                rs += stage_val<CODE>(st, j0 + k * G, sdict) * ((c[k] == row) ? xn : xv[k]);
                    }
                    if (G > 1) rs = group_sum<G>(rs);
                    if (active && sub == 0) tile_row_residual(a, row, st.bseg[row - voff], rs, r2);
                }
            }
        } else {
            // a single row longer than a tile: the whole warp strides over it in global memory
            const int row = row0;
            double sum = 0.0, diag = 0.0;
            int jd = -1;
            for (int jj = s0 + lane; jj < s0 + len; jj += 32) {
                int c;
                double v;
                global_entry<CODE>(a, jj, row, sdict, c, v);
                const double xv = (OP == OP_GS) ? a.x[c < 0 ? 0 : c] : __ldg(a.x + c);
                if (kNeedDiag && c == row) { diag = v; jd = jj; }
                else if (OP != OP_GS || c >= 0) sum += v * xv;
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
                    const double g = (a.b[row] - sum) / diag;
                    a.y[row] = (a.omega == 1.0) ? g : a.omega * g + (1.0 - a.omega) * a.y[row];
                }
            }
            if (OP == OP_GS && a.r != nullptr) {          // last-wave residual, as in the tile path above
                __syncwarp();
                const double xn = __shfl_sync(0xffffffffu, lane == 0 ? a.y[row] : 0.0, 0);
                double rs = 0.0;
                for (int jj = s0 + lane; jj < s0 + len; jj += 32) {
                    int c;
                    double v;
                    global_entry<CODE>(a, jj, row, sdict, c, v);
                    rs += v * ((c == row) ? xn : a.x[c]);
                }
                rs = group_sum<32>(rs);
                if (lane == 0) { const double r = a.b[row] - rs; a.r[row] = r; r2 += r * r; }
            }
        }
        __syncwarp();             // every lane is done with this stage before the TMA refills it
        stage = (stage + 1) % STAGES;
    }
    if ((OP == OP_RESID || OP == OP_JACOBI || OP == OP_GS) && a.partials != nullptr) {
        const double tsum = block_sum<C::WARPS * 32>(r2);
        if (threadIdx.x == 0) a.partials[blockIdx.x] = tsum;
    }
}

// The CTA's copy of a row-coded operator's tables: pair values and column offsets apart, so that a batch of gathers
// holds only the offsets it needs to issue them and the values are read when the products are summed
struct RowCodeSmem {
    double v[kMaxCodes];
    int delta[kMaxCodes];
    RowPattern pat[kMaxCodes];
};

// Gathers a row-coded row issues back to back: batches of this many entries keep the kernel within the registers of
// kTileCtas resident CTAs per SM
constexpr int kRowCodeBatch = 4;

// Entries k0 .. min(k0 + kRowCodeBatch, len) - 1 of a row-coded row, gathers issued back to back, then
// sum += v * x[c] in stored order with the diagonal (Jacobi, Gauss-Seidel) kept apart: csr_tile_kernel's G = 1 step
template <int OP>
__device__ __forceinline__ void row_code_sum(const TileArgs &a, const RowCodeSmem &sm, const RowPattern &pt, int k0,
                                             int len, int row, unsigned long long pol_last, double &sum, double &diag)
{
    constexpr bool kNeedDiag = (OP == OP_JACOBI || OP == OP_GS);
    constexpr int kN = kRowCodeBatch;
    double xv[kN];
#pragma unroll
    for (int kk = 0; kk < kN; kk++) {
        const int k = k0 + kk;
        xv[kk] = 0.0;
        if (k < kRowCodeMaxLen && k < len) {
            const int c = row + sm.delta[pt.pair[k]];
            if (!(kNeedDiag && c == row) && (OP != OP_GS || c >= 0)) {   // zero-start padding (c = -1): no term
                if (a.hints) xv[kk] = (OP == OP_GS) ? ld_x_hint(a.x + c, pol_last) : ld_x_hint_nc(a.x + c, pol_last);
                else xv[kk] = (OP == OP_GS) ? a.x[c] : __ldg(a.x + c);
            }
        }
    }
#pragma unroll
    for (int kk = 0; kk < kN; kk++) {
        const int k = k0 + kk;
        if (k < kRowCodeMaxLen && k < len) {
            const unsigned e = pt.pair[k];
            const int c = row + sm.delta[e];
            const double v = sm.v[e];
            if (kNeedDiag && c == row) diag = v;
            else if (OP != OP_GS || c >= 0) sum += v * xv[kk];
        }
    }
}

// The same entries for the residual of a sweep's last Gauss-Seidel wave: the row's new x_i where it reads itself
__device__ __forceinline__ void row_code_resid(const TileArgs &a, const RowCodeSmem &sm, const RowPattern &pt, int k0,
                                               int len, int row, double xn, unsigned long long pol_last, double &rs)
{
    constexpr int kN = kRowCodeBatch;
    double xv[kN];
#pragma unroll
    for (int kk = 0; kk < kN; kk++) {
        const int k = k0 + kk;
        xv[kk] = xn;
        if (k < kRowCodeMaxLen && k < len) {
            const int c = row + sm.delta[pt.pair[k]];
            if (c != row) xv[kk] = a.hints ? ld_x_hint(a.x + c, pol_last) : a.x[c];
        }
    }
#pragma unroll
    for (int kk = 0; kk < kN; kk++) {
        const int k = k0 + kk;
        if (k < kRowCodeMaxLen && k < len) rs += sm.v[pt.pair[k]] * xv[kk];
    }
}

// Row-coded tile-list kernel (one lane per row): tile t -> warp t mod #warps of the persistent grid, row row0 + lane
// (+ 32 on a tile's second pass) -> lane, as csr_tile_kernel<1, OP, C> assigns them, so each lane sums the same rows
// in the same order and the |r|^2 partials are the same.  Row i's entries are pairs[patterns[codes[i]].pair[k]], k in
// stored order; both tables sit in shared memory.  The row codes of tile t + #warps are loaded before tile t is
// reduced, and its descriptor one tile earlier still; b and the old x are loaded with the row's gathers.
template <int OP, class C>
__global__ void __launch_bounds__(C::WARPS * 32, kTileCtas[OP]) csr_rowcode_kernel(const TileArgs a)
{
    __shared__ RowCodeSmem sm;
    for (int i = threadIdx.x; i < a.ndict; i += blockDim.x) {
        sm.v[i] = a.pairs[i].v;
        sm.delta[i] = a.pairs[i].delta;
    }
    for (int i = threadIdx.x; i < kMaxCodes; i += blockDim.x) sm.pat[i] = a.patterns[i];
    __syncthreads();
    constexpr bool kB = (OP == OP_RESID || OP == OP_JACOBI || OP == OP_GS);
    constexpr bool kX = (OP == OP_JACOBI);
    constexpr int kPass = C::RMAX / 32;             // G = 1: 32 rows per pass
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned long long pol_last = policy_evict_last();
    const int nwarps = gridDim.x * C::WARPS;
    int t = a.tile_begin + blockIdx.x * C::WARPS + warp;
    double r2 = 0.0;

    // row codes of one tile (rows row0 .. row0 + nrows): pass p's code -> byte p of `code`, row row0 + 32 p + lane
    auto fetch = [&](int r0, int nr) {
        unsigned code = 0;
#pragma unroll
        for (int p = 0; p < kPass; p++)
            if (p * 32 + lane < nr) code |= (unsigned)__ldg(a.codes + r0 + p * 32 + lane) << (8 * p);
        return code;
    };
    int row0 = 0, nrows = 0, nrow0 = 0, nnrows = 0;     // this tile and tile t + nwarps
    unsigned code = 0;
    if (t < a.tile_end) {
        row0 = a.tiles[t].row0;
        nrows = a.tiles[t + 1].row0 - row0;
        code = fetch(row0, nrows);
        if (t + nwarps < a.tile_end) {
            nrow0 = a.tiles[t + nwarps].row0;
            nnrows = a.tiles[t + nwarps + 1].row0 - nrow0;
        }
    }
    for (; t < a.tile_end; t += nwarps) {
        const unsigned ncode = fetch(nrow0, t + nwarps < a.tile_end ? nnrows : 0);
        const int trow0 = nrow0, tnrows = nnrows;
        if (t + 2 * nwarps < a.tile_end) {
            nrow0 = a.tiles[t + 2 * nwarps].row0;
            nnrows = a.tiles[t + 2 * nwarps + 1].row0 - nrow0;
        }
#pragma unroll 1
        for (int p = 0; p < kPass; p++) {
            if (p * 32 >= nrows) break;
            const bool active = p * 32 + lane < nrows;
            const int row = row0 + p * 32 + lane;
            const double bi = (kB && active) ? __ldg(a.b + row) : 0.0;     // in flight with the gathers below
            const double xi = (kX && active) ? a.x[row] : 0.0;
            const RowPattern &pt = sm.pat[(code >> (8 * p)) & 0xffu];
            const int len = active ? pt.len : 0;
            double sum = 0.0, diag = 0.0;
            // the entries in batches of gathers, each issued back to back; the products are summed in stored order
#pragma unroll
            for (int k0 = 0; k0 < kRowCodeMaxLen; k0 += kRowCodeBatch)
                if (k0 < len) row_code_sum<OP>(a, sm, pt, k0, len, row, pol_last, sum, diag);
            double xn = 0.0;
            if (active) xn = tile_row_epilogue<OP>(a, row, sum, diag, [&] { return bi; }, [&] { return xi; }, r2);
            if (OP == OP_GS && a.r != nullptr) {
                // the last wave's residual, as csr_tile_kernel forms it: the new x_i where the row reads itself
                double rs = 0.0;
#pragma unroll
                for (int k0 = 0; k0 < kRowCodeMaxLen; k0 += kRowCodeBatch)
                    if (k0 < len) row_code_resid(a, sm, pt, k0, len, row, xn, pol_last, rs);
                if (active) tile_row_residual(a, row, bi, rs, r2);
            }
        }
        row0 = trow0;
        nrows = tnrows;
        code = ncode;
    }
    if (kB && a.partials != nullptr) {
        const double tsum = block_sum<C::WARPS * 32>(r2);
        if (threadIdx.x == 0) a.partials[blockIdx.x] = tsum;
    }
}

}  // namespace amgb
