// engine.cu -- H100-native AMG solve-phase engine: hierarchy in HBM, cycle driver, C ABI.
//
// Replaces (paths relative to the reference tree):
//   pyamg/multilevel.py:398-582   MultilevelSolver.solve      -> amgb_solve
//   pyamg/multilevel.py:584-662   MultilevelSolver.__solve    -> Engine::cycle (V/W/F, captured as CUDA graphs)
//   pyamg/multilevel.py:717-721   'pinv' coarse solver apply   -> dense_matvec_kernel
//   pyamg/relaxation/relaxation.py + pyamg/amg_core/relaxation.h sweeps -> csr_kernels.cuh
//   scipy csr_matvec/bsr_matvec call sites multilevel.py:545,567,612,614,660 -> csr_rows_kernel<...>
//
// Design: one process per GPU; every operator of the hierarchy lives in HBM as int32/fp64 CSR
// (BSR blocks are expanded to point CSR at upload: same per-row summation order as bsr_matvec);
// all level vectors are preallocated; a cycle is a fixed launch sequence, captured once per
// cycle type into a CUDA graph so that the launch-latency-bound coarse levels cost ~1 graph node
// each instead of a Python round trip.  No CPU fallback anywhere.
#include "../../include/pyamg_b200.h"
#include "csr_kernels.cuh"
#include "tile_kernels.cuh"
#ifndef AMGB_EMU
#include <cuda_profiler_api.h>
#endif
#include <array>
#include "tail_kernel.cuh"
#include "grid_kernel.cuh"
#include "coloring.cuh"
#include "resident_kernel.cuh"
#include "tile_flat_kernel.cuh"
#include "multi_rhs_kernels.cuh"
#include "spgemm.cuh"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

using namespace amgb;

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;

static int fail(int code, const std::string &msg)
{
    g_err = msg;
    return code;
}

#define CK(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return fail(AMGB_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_) +      \
                                        " (" __FILE__ ":" + std::to_string(__LINE__) + ")");  \
    } while (0)

#define RET(call)                 \
    do {                          \
        int rc_ = (call);         \
        if (rc_ != AMGB_OK) return rc_; \
    } while (0)

extern "C" const char *amgb_last_error(void) { return g_err.c_str(); }
extern "C" int amgb_version(void) { return 101; }
extern "C" int amgb_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

// ------------------------------------------------------------------------------------------
// launch settings
// ------------------------------------------------------------------------------------------
// Every AMGB_* switch of the engine and the device properties its launches are sized from, filled once by
// read_settings.  A hierarchy keeps the settings it was created under; the entries without a hierarchy (amgb_dev_*,
// the amgb_host_* helpers that launch) read them for the current device at each call.  The launch helpers take them
// as an argument, so hierarchies built under different settings or on different devices can be used side by side.
struct Settings {
    int num_sms = 0;               // SM count of the device (132 on an H100 SXM)
    int lanes = 0;                 // AMGB_LANES: lanes per row of the rows kernel (0: from the mean row length)
    int tile_G = 0;                // AMGB_TILE_G: lanes per row of the tile kernel (0: from the mean row length)
    double lane_entries = 12.0;    // AMGB_TILE_LANE_ENTRIES: tile lanes per row G double while mean row length > this * G
    bool pdl = true;               // AMGB_NO_PDL=1: plain stream-ordered launches for the lanes-per-row kernel
    int tile_cfg = 6;              // AMGB_TILE_CFG: which TileCfg geometry (tile_kernels.cuh)
    int tile_ctas[5] = {2, 2, 2, 2, 2};   // resident CTAs per SM of csr_tile_kernel<*, OP, cfg>, per OP (AMGB_TILE_CTAS caps it)
    int tile_T = 256, tile_rmax = 64, tile_warps = 8;
    int tile_hints = 1;            // AMGB_NO_HINTS=1 disables the L2 eviction hints
    bool tile_pdl = false;         // AMGB_TILE_PDL=1 (experimental): programmatic dependent launch of the tile kernel
    int tile_flat = 0;             // AMGB_TILE_FLAT=1 (experimental): flat-gather tile kernel (tile_flat_kernel.cuh); 2: only R (all levels) and P (levels >= 1)
    // second geometry for the denser operators of a hierarchy (mean row length above dense_avg): AMGB_TILE_DENSE_CFG=7
    int dense_cfg = 0;
    double dense_avg = 12.0;
    int dense_ctas[5] = {2, 2, 2, 2, 2};
    int dense_T = 352, dense_rmax = 64;

    bool use_graph = true;         // AMGB_NO_GRAPH=1: every cycle issued launch by launch
    bool use_tiles = true;         // AMGB_NO_TILES=1: the lanes-per-row kernel only
    bool use_permute = true;       // AMGB_NO_PERMUTE=1: no wave-major (or C|F) row layouts
    bool use_cf_layout = true;     // AMGB_NO_CF_LAYOUT=1: CF / FC Jacobi through row lists on the natural numbering
    bool use_resident = false;     // AMGB_RESIDENT=1: experimental DSMEM-resident Gauss-Seidel applications
    long long resident_max_rows = 65536;   // AMGB_RESIDENT_MAX_ROWS
    bool use_wave_resid = true;    // AMGB_NO_WAVE_RESID=1: the residual after a Gauss-Seidel smoother as one separate launch
    bool use_zero_start = true;    // AMGB_NO_ZERO_START=1: no zero-start copies; coarse pre-smoothers stream the full operator
    bool use_value_codes = true;   // AMGB_NO_VALUE_CODES=1: level operators stream fp64 values on every tile launch
    bool use_pair_codes = true;    // AMGB_NO_PAIR_CODES=1: no pair codes; operators that would get them get value codes
    bool use_row_codes = true;     // AMGB_NO_ROW_CODES=1: operators that would get row codes keep per-entry pair codes
    long long tile_min_nnz = 1500000;      // AMGB_TILE_MIN_NNZ: smaller launches use the lanes-per-row kernel
    // AMGB_PAIR_MIN_NNZ: smaller operators keep value codes.  The default is the default tile threshold, below which
    // launches go to the rows kernel, so by default it excludes nothing that would stream tiles; with AMGB_TILE_MIN_NNZ
    // lowered (tests, tuning sweeps) small operators keep the value-code launches and accounting they had.  0: every
    // operator that qualifies gets pair codes.
    long long pair_min_nnz = 1500000;
    // AMGB_ROW_MIN_NNZ: smaller operators keep per-entry pair codes (default: the default tile threshold, as
    // AMGB_PAIR_MIN_NNZ).  Its own knob, so that small operators can be pair-coded without being row-coded.
    long long row_min_nnz = 1500000;

    // coarse tail (tail_kernel.cuh, grid_kernel.cuh)
    bool tail_grid = false;        // AMGB_TAIL_GRID=1: the grid mode, one cooperatively launched CTA per SM
    // AMGB_TAIL_NNZ: levels with at most this many entries run in the tail.  Default 0 = off: with programmatic
    // dependent launch the per-wave launches of a CUDA graph pipeline the small levels; the tail remains selectable.
    // The grid mode's default is ~12 M entries (L2-resident waves); AMGB_NO_TAIL=1: -1, no level runs in the tail.
    long long tail_nnz_limit = 0;
    double tail_solo_bytes = 400000.0;     // AMGB_TAIL_SOLO_BYTES: steps moving at most this much run on one CTA
    int tail_cluster = 16;         // AMGB_TAIL_CLUSTER: largest cluster of the cluster tail kernel
    int grid_ctas = 0;             // AMGB_GRID_CTAS: CTAs of the grid mode (default and at most: one per SM)

    bool verbose = false;          // AMGB_VERBOSE=1: the tile streams and the coarse tail of a new hierarchy on stderr
    std::vector<std::array<long long, 3>> ncu_select;   // AMGB_NCU_SELECT, counted down by amgb_hierarchy::ncu_gate_begin
};

template <class C>
static void tile_cfg_ctas(size_t smem_per_sm, int ctas_cap, int *ctas)
{
    const size_t smem[5] = {tile_smem_bytes<C, OP_SPMV>(), tile_smem_bytes<C, OP_RESID>(), tile_smem_bytes<C, OP_PADD>(),
                            tile_smem_bytes<C, OP_JACOBI>(), tile_smem_bytes<C, OP_GS>()};
    for (int op = OP_SPMV; op <= OP_GS; op++) {
        int c = std::max(1, (int)(smem_per_sm / (smem[op] + 1024)));
        c = std::min(c, 2048 / (C::WARPS * 32));
        // per-epilogue cap on resident CTAs (tools/microbench.py, 256^3 7-point): resident warps hide the
        // gather latency, but the shared memory they pin shrinks L1 -- the sweet spot depends on the stage size.
        // Tuned on the previous target (also 228 KB of shared memory per SM) and carried over, not re-tuned for H100
        const int cap = ctas_cap > 0 ? ctas_cap : kTileCtas[op];
        ctas[op] = std::max(1, std::min(c, cap));
    }
}

template <class C>
static void tile_cfg_select(Settings &S, size_t smem_per_sm, int ctas_cap)
{
    S.tile_T = C::T;
    S.tile_rmax = C::RMAX;
    S.tile_warps = C::WARPS;
    tile_cfg_ctas<C>(smem_per_sm, ctas_cap, S.tile_ctas);
}

// The only reader of the AMGB_* environment (besides amgb_comm_create's AMGB_COMM_*): fills a fresh S for `device`
static int read_settings(int device, Settings &S)
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    S.num_sms = prop.multiProcessorCount;
    auto flag = [](const char *name) { const char *v = getenv(name); return v && v[0] == '1'; };
    auto lanes = [](const char *name) {
        const char *v = getenv(name);
        const int g = v ? atoi(v) : 0;
        return (g == 1 || g == 2 || g == 4 || g == 8 || g == 16 || g == 32) ? g : 0;
    };
    S.lanes = lanes("AMGB_LANES");
    S.tile_G = lanes("AMGB_TILE_G");

    const char *c = getenv("AMGB_TILE_CTAS");
    const int ctas_cap = (c && atoi(c) >= 1) ? atoi(c) : 0;   // 0 = per-epilogue default cap (kTileCtas)
    const char *e = getenv("AMGB_TILE_CFG");
    S.tile_cfg = e ? atoi(e) : 6;   // default geometry (tools/tune_tiles.py compares the others)
    switch (S.tile_cfg) {
    case 0: tile_cfg_select<TileCfg0>(S, prop.sharedMemPerMultiprocessor, ctas_cap); break;
    case 1: tile_cfg_select<TileCfg1>(S, prop.sharedMemPerMultiprocessor, ctas_cap); break;
    case 4: tile_cfg_select<TileCfg4>(S, prop.sharedMemPerMultiprocessor, ctas_cap); break;
    default: S.tile_cfg = 6; tile_cfg_select<TileCfg6>(S, prop.sharedMemPerMultiprocessor, ctas_cap); break;
    }
    S.tile_hints = !flag("AMGB_NO_HINTS");
    S.pdl = !flag("AMGB_NO_PDL");
    S.tile_pdl = flag("AMGB_TILE_PDL");
    const char *tf = getenv("AMGB_TILE_FLAT");
    // defaults: flat gathers for the restrictions and the coarse prolongations (mode 2) and the second, larger tile
    // geometry for operators with more than ~12 entries per row.  AMGB_TILE_FLAT=0 / AMGB_TILE_DENSE_CFG=0 switch
    // them off.
    const int flat_mode = tf ? ((tf[0] == '1' || tf[0] == '2') ? (tf[0] - '0') : 0) : 2;
    S.tile_flat = (S.tile_cfg == 6) ? flat_mode : 0;     // default geometry only
    const char *dc = getenv("AMGB_TILE_DENSE_CFG");
    S.dense_cfg = dc ? ((atoi(dc) == 7) ? 7 : 0) : 7;
    if (S.dense_cfg == 7) {
        S.dense_T = TileCfg7::T; S.dense_rmax = TileCfg7::RMAX;
        tile_cfg_ctas<TileCfg7>(prop.sharedMemPerMultiprocessor, ctas_cap, S.dense_ctas);
    }
    const char *da = getenv("AMGB_TILE_DENSE_AVG");
    S.dense_avg = (da && atof(da) > 0) ? atof(da) : 12.0;
    const char *le = getenv("AMGB_TILE_LANE_ENTRIES");
    S.lane_entries = (le && atof(le) >= 1.0) ? atof(le) : 12.0;

    S.use_graph = !flag("AMGB_NO_GRAPH");
    S.use_tiles = !flag("AMGB_NO_TILES");
    S.use_permute = !flag("AMGB_NO_PERMUTE");
    S.use_cf_layout = !flag("AMGB_NO_CF_LAYOUT");
    S.use_resident = flag("AMGB_RESIDENT");
    S.use_wave_resid = !flag("AMGB_NO_WAVE_RESID");
    S.use_zero_start = !flag("AMGB_NO_ZERO_START");
    S.use_value_codes = !flag("AMGB_NO_VALUE_CODES");
    S.use_pair_codes = !flag("AMGB_NO_PAIR_CODES");
    S.use_row_codes = !flag("AMGB_NO_ROW_CODES");
    if (const char *v = getenv("AMGB_RESIDENT_MAX_ROWS")) S.resident_max_rows = atoll(v);
    if (const char *tm = getenv("AMGB_TILE_MIN_NNZ"))
        if (atoll(tm) >= 0) S.tile_min_nnz = atoll(tm);
    if (const char *pm = getenv("AMGB_PAIR_MIN_NNZ"))
        if (atoll(pm) >= 0) S.pair_min_nnz = atoll(pm);
    if (const char *rm = getenv("AMGB_ROW_MIN_NNZ"))
        if (atoll(rm) >= 0) S.row_min_nnz = atoll(rm);

    S.tail_grid = flag("AMGB_TAIL_GRID");
    if (S.tail_grid) S.tail_nnz_limit = 12000000;
    const char *tn = getenv("AMGB_TAIL_NNZ");
    if (tn && atoll(tn) >= 0) S.tail_nnz_limit = atoll(tn);
    if (flag("AMGB_NO_TAIL")) S.tail_nnz_limit = -1;
    if (const char *sb = getenv("AMGB_TAIL_SOLO_BYTES")) S.tail_solo_bytes = atof(sb);
    if (const char *cs = getenv("AMGB_TAIL_CLUSTER")) S.tail_cluster = atoi(cs);
    const char *gc = getenv("AMGB_GRID_CTAS");
    S.grid_ctas = (gc && atoi(gc) >= 1) ? std::min(atoi(gc), S.num_sms) : S.num_sms;

    S.verbose = flag("AMGB_VERBOSE");
    if (const char *ns = getenv("AMGB_NCU_SELECT")) {
        std::string str(ns);
        size_t pos = 0;
        while (pos < str.size()) {
            size_t end = str.find(',', pos);
            if (end == std::string::npos) end = str.size();
            long long l = 0, o = 0, n = 0;
            if (sscanf(str.substr(pos, end - pos).c_str(), "%lld:%lld:%lld", &l, &o, &n) == 3)
                S.ncu_select.push_back({l, o, n});
            pos = end + 1;
        }
    }
    return AMGB_OK;
}

// S = the settings of the entries without a hierarchy on the current device, read at their first call there:
// cudaGetDeviceProperties alone takes milliseconds, far longer than the launches these entries make
constexpr int kMaxDevices = 64;
static int current_settings(Settings &S)
{
    int device = 0;
    CK(cudaGetDevice(&device));
    if (device >= kMaxDevices) return read_settings(device, S);
    static std::mutex mu;
    static Settings cached[kMaxDevices];
    std::lock_guard<std::mutex> lock(mu);
    if (cached[device].num_sms == 0) RET(read_settings(device, cached[device]));   // 0: not read yet
    S = cached[device];
    return AMGB_OK;
}

// ------------------------------------------------------------------------------------------
// launch helpers
// ------------------------------------------------------------------------------------------
static int pick_lanes(const Settings &S, long long nnz, long long n_rows)
{
    if (S.lanes != 0) return S.lanes;
    if (n_rows <= 0) return 4;
    const double avg = (double)nnz / (double)n_rows;
    int g = 2;
    while (g < 32 && (double)g < avg) g <<= 1;   // smallest power of two >= mean row length
    return g;
}

static inline long long csr_grid(long long n, int lanes)
{
    return (n * lanes + kCsrThreads - 1) / kCsrThreads;
}

// grid of the grid-stride vector kernels: 256 threads per block, at most 16 blocks per SM
static inline unsigned vec_grid(const Settings &S, long long n)
{
    return (unsigned)std::max<long long>(1, std::min<long long>((n + 255) / 256, (long long)S.num_sms * 16));
}

// cudaFuncSetAttribute acts on the current device's copy of a kernel, so the opt-in to more than 48 KB of dynamic
// shared memory is remembered per device ordinal in `done` (kMaxDevices flags; devices past that opt in at every
// launch).  Two threads setting the same attribute to the same value is harmless.
static int optin_smem(const void *kernel, size_t smem, std::atomic<bool> *done)
{
    int device = 0;
    CK(cudaGetDevice(&device));
    const bool known = device < kMaxDevices;
    if (known && done[device].load(std::memory_order_relaxed)) return AMGB_OK;
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (known) done[device].store(true, std::memory_order_relaxed);
    return AMGB_OK;
}

template <int G, int OP, bool INDEXED>
static int launch_rows_one(const Settings &S, const CsrRowArgs &a, unsigned grid, cudaStream_t s)
{
    if (!S.pdl) {
        csr_rows_kernel<G, OP, INDEXED><<<grid, kCsrThreads, 0, s>>>(a);
        return AMGB_OK;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kCsrThreads);
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    CK(cudaLaunchKernelEx(&cfg, csr_rows_kernel<G, OP, INDEXED>, a));
    return AMGB_OK;
}

template <int OP, bool INDEXED>
static int launch_csr_g(const Settings &S, int lanes, const CsrRowArgs &a, cudaStream_t s)
{
    if (a.n <= 0) return AMGB_OK;
    const long long grid = csr_grid(a.n, lanes);
    if (grid > 2147483647LL) return fail(AMGB_EINVAL, "launch grid too large");
    const unsigned g = (unsigned)grid;
    switch (lanes) {
    case 1: RET((launch_rows_one<1, OP, INDEXED>(S, a, g, s))); break;
    case 2: RET((launch_rows_one<2, OP, INDEXED>(S, a, g, s))); break;
    case 4: RET((launch_rows_one<4, OP, INDEXED>(S, a, g, s))); break;
    case 8: RET((launch_rows_one<8, OP, INDEXED>(S, a, g, s))); break;
    case 16: RET((launch_rows_one<16, OP, INDEXED>(S, a, g, s))); break;
    case 32: RET((launch_rows_one<32, OP, INDEXED>(S, a, g, s))); break;
    default: return fail(AMGB_EINVAL, "lanes must be a power of two in 1..32");
    }
    CK(cudaGetLastError());
    return AMGB_OK;
}

static int launch_csr(const Settings &S, int op, int lanes, const CsrRowArgs &a, cudaStream_t s)
{
    const bool idx = a.rows != nullptr;
    switch (op) {
    case OP_SPMV: return idx ? launch_csr_g<OP_SPMV, true>(S, lanes, a, s) : launch_csr_g<OP_SPMV, false>(S, lanes, a, s);
    case OP_RESID: return idx ? launch_csr_g<OP_RESID, true>(S, lanes, a, s) : launch_csr_g<OP_RESID, false>(S, lanes, a, s);
    case OP_PADD: return idx ? launch_csr_g<OP_PADD, true>(S, lanes, a, s) : launch_csr_g<OP_PADD, false>(S, lanes, a, s);
    case OP_JACOBI: return idx ? launch_csr_g<OP_JACOBI, true>(S, lanes, a, s) : launch_csr_g<OP_JACOBI, false>(S, lanes, a, s);
    case OP_GS: return idx ? launch_csr_g<OP_GS, true>(S, lanes, a, s) : launch_csr_g<OP_GS, false>(S, lanes, a, s);
    }
    return fail(AMGB_EINVAL, "unknown csr op");
}

static int launch_fill(const Settings &S, double *x, long long n, double v, cudaStream_t s)
{
    if (n <= 0) return AMGB_OK;
    fill_kernel<<<vec_grid(S, n), 256, 0, s>>>(x, n, v);
    CK(cudaGetLastError());
    return AMGB_OK;
}

// two-stage reductions (norms, dot products): a fixed grid of 8 blocks per SM -> deterministic partial sums
// (the partials buffer holds kSumsqBlocks = 148 x 8, enough for any device of up to 148 SMs)
static inline int sumsq_blocks(const Settings &S) { return std::min(kSumsqBlocks, S.num_sms * 8); }

// ------------------------------------------------------------------------------------------
// tile-kernel launch
// ------------------------------------------------------------------------------------------
// pair-coded kernels exist for G <= kPairMaxG lanes per row and without programmatic launch only (upload_csr gives
// pair codes to no other launch geometry): the 5- to 27-point stencils that have few enough pairs need G <= 4
constexpr int kPairMaxG = 4;

template <int OP, class C, int CODE = CODE_NONE>
static int launch_tile_cfg(const Settings &S, int G, const TileArgs &a, int grid, cudaStream_t s)
{
    const dim3 g((unsigned)grid), b(C::WARPS * 32);
    constexpr size_t smem = tile_smem_bytes<C, OP, CODE>();
#define AMGB_TILE_CASE(GG)                                                                               \
    case GG: {                                                                                           \
        if constexpr (CODE == CODE_PAIR8 && GG > kPairMaxG) {                                            \
            return fail(AMGB_EINVAL, "tile kernel: no pair-coded kernel for this many lanes per row");   \
        } else {                                                                                         \
        if constexpr (std::is_same<C, TileCfg6>::value && CODE != CODE_PAIR8) {                          \
            if (S.tile_pdl) {   /* opt-in: programmatic dependent launch, default geometry only */      \
                static std::atomic<bool> pdl_attr_done[kMaxDevices];                                     \
                RET(optin_smem((const void *)csr_tile_kernel<GG, OP, C, true, CODE>, smem, pdl_attr_done)); \
                cudaLaunchConfig_t cfg = {};                                                             \
                cfg.gridDim = g; cfg.blockDim = b; cfg.dynamicSmemBytes = smem; cfg.stream = s;          \
                cudaLaunchAttribute at[1];                                                               \
                at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                           \
                at[0].val.programmaticStreamSerializationAllowed = 1;                                    \
                cfg.attrs = at; cfg.numAttrs = 1;                                                        \
                CK(cudaLaunchKernelEx(&cfg, csr_tile_kernel<GG, OP, C, true, CODE>, a));                \
                break;                                                                                   \
            }                                                                                            \
        }                                                                                                \
        static std::atomic<bool> attr_done[kMaxDevices];                                                 \
        RET(optin_smem((const void *)csr_tile_kernel<GG, OP, C, false, CODE>, smem, attr_done));         \
        csr_tile_kernel<GG, OP, C, false, CODE><<<g, b, smem, s>>>(a);                                   \
        break;                                                                                           \
        }                                                                                                \
    }
    switch (G) {
        AMGB_TILE_CASE(1)
        AMGB_TILE_CASE(2)
        AMGB_TILE_CASE(4)
        AMGB_TILE_CASE(8)
        AMGB_TILE_CASE(16)
        AMGB_TILE_CASE(32)
    default: return fail(AMGB_EINVAL, "tile kernel: G must be a power of two in 1..32");
    }
#undef AMGB_TILE_CASE
    CK(cudaGetLastError());
    return AMGB_OK;
}

// row-coded kernel: one lane per row, tiles of the default or the dense geometry (upload_csr), which share the warps
// per CTA and the rows per tile that csr_rowcode_kernel takes from TileCfg6
static_assert(TileCfg6::WARPS == TileCfg7::WARPS && TileCfg6::RMAX == TileCfg7::RMAX, "row-coded tile geometry");
template <int OP>
static int launch_rowcode(int G, const TileArgs &a, int grid, cudaStream_t s)
{
    if (G != 1) return fail(AMGB_EINVAL, "tile kernel: no row-coded kernel for more than one lane per row");
    csr_rowcode_kernel<OP, TileCfg6><<<dim3((unsigned)grid), dim3(TileCfg6::WARPS * 32), 0, s>>>(a);
    CK(cudaGetLastError());
    return AMGB_OK;
}

template <int OP>
static int launch_tile_op(const Settings &S, int G, const TileArgs &a, int grid, cudaStream_t s, int cfg)
{
    if (a.pairs != nullptr && a.patterns != nullptr) return launch_rowcode<OP>(G, a, grid, s);   // row codes: G = 1
    if (a.pairs != nullptr) {        // pair codes: the default and the dense geometry, G <= kPairMaxG (upload_csr)
        if (cfg == 7) return launch_tile_cfg<OP, TileCfg7, CODE_PAIR8>(S, G, a, grid, s);
        if (S.tile_cfg == 6) return launch_tile_cfg<OP, TileCfg6, CODE_PAIR8>(S, G, a, grid, s);
        return fail(AMGB_EINVAL, "tile kernel: no pair-coded kernel for this tile geometry");
    }
    if (a.codes != nullptr) {        // value codes: built for the default and the dense geometry only (upload_csr)
        if (cfg == 7) return launch_tile_cfg<OP, TileCfg7, CODE_VAL8>(S, G, a, grid, s);
        if (S.tile_cfg == 6) return launch_tile_cfg<OP, TileCfg6, CODE_VAL8>(S, G, a, grid, s);
        return fail(AMGB_EINVAL, "tile kernel: no value-coded kernel for this tile geometry");
    }
    if (cfg == 7) return launch_tile_cfg<OP, TileCfg7>(S, G, a, grid, s);
    switch (S.tile_cfg) {
    case 0: return launch_tile_cfg<OP, TileCfg0>(S, G, a, grid, s);
    case 1: return launch_tile_cfg<OP, TileCfg1>(S, G, a, grid, s);
    case 4: return launch_tile_cfg<OP, TileCfg4>(S, G, a, grid, s);
    default: return launch_tile_cfg<OP, TileCfg6>(S, G, a, grid, s);
    }
}

// flat-gather variant (G == 0 in DevCsr::tile_G): default geometry, with or without programmatic launch
template <int OP, bool PDL, bool CODED>
static int launch_tile_flat_one(const TileArgs &a, int grid, cudaStream_t s)
{
    using C = TileCfg6;
    constexpr size_t smem = tile_flat_smem_bytes<C, OP, CODED>();
    static std::atomic<bool> attr_done[kMaxDevices];
    RET(optin_smem((const void *)csr_tile_flat_kernel<OP, C, PDL, CODED>, smem, attr_done));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(C::WARPS * 32); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = PDL ? 1 : 0;
    CK(cudaLaunchKernelEx(&cfg, csr_tile_flat_kernel<OP, C, PDL, CODED>, a));
    return AMGB_OK;
}
template <int OP>
static int launch_tile_flat(const Settings &S, const TileArgs &a, int grid, cudaStream_t s)
{
    if (a.pairs != nullptr) return fail(AMGB_EINVAL, "flat tile kernel: no pair-coded variant");
    if (a.codes != nullptr)
        return S.tile_pdl ? launch_tile_flat_one<OP, true, true>(a, grid, s) : launch_tile_flat_one<OP, false, true>(a, grid, s);
    return S.tile_pdl ? launch_tile_flat_one<OP, true, false>(a, grid, s) : launch_tile_flat_one<OP, false, false>(a, grid, s);
}

static int launch_tile(const Settings &S, int op, int G, TileArgs a, int grid, cudaStream_t s, int cfg = 0)
{
    if (a.tile_end <= a.tile_begin) return AMGB_OK;
    a.hints = S.tile_hints;
    if (G == 0) {
        switch (op) {
        case OP_SPMV: return launch_tile_flat<OP_SPMV>(S, a, grid, s);
        case OP_RESID: return launch_tile_flat<OP_RESID>(S, a, grid, s);
        case OP_PADD: return launch_tile_flat<OP_PADD>(S, a, grid, s);
        case OP_JACOBI: return launch_tile_flat<OP_JACOBI>(S, a, grid, s);
        case OP_GS: return launch_tile_flat<OP_GS>(S, a, grid, s);
        }
        return fail(AMGB_EINVAL, "unknown tile op");
    }
    switch (op) {
    case OP_SPMV: return launch_tile_op<OP_SPMV>(S, G, a, grid, s, cfg);
    case OP_RESID: return launch_tile_op<OP_RESID>(S, G, a, grid, s, cfg);
    case OP_PADD: return launch_tile_op<OP_PADD>(S, G, a, grid, s, cfg);
    case OP_JACOBI: return launch_tile_op<OP_JACOBI>(S, G, a, grid, s, cfg);
    case OP_GS: return launch_tile_op<OP_GS>(S, G, a, grid, s, cfg);
    }
    return fail(AMGB_EINVAL, "unknown tile op");
}

static inline int tile_grid(const Settings &S, int op, int ntiles, int cfg = 0)
{
    const int full = S.num_sms * (cfg == 7 ? S.dense_ctas[op] : S.tile_ctas[op]);
    const int need = (ntiles + S.tile_warps - 1) / S.tile_warps;
    return std::max(1, std::min(full, need));
}

// ------------------------------------------------------------------------------------------
// host / device containers
// ------------------------------------------------------------------------------------------
struct HostCsr {   // point CSR on the host (BSR already expanded)
    int n_rows = 0, n_cols = 0;
    std::vector<int> Ap, Aj;
    std::vector<double> Ax;
};

struct DevCsr {
    int n_rows = 0, n_cols = 0;
    long long nnz = 0;
    int *Ap = nullptr, *Aj = nullptr;
    double *Ax = nullptr;
    int lanes = 8;               // rows kernel: lanes per row
    // tile kernel
    TileDesc *tiles = nullptr;   // n_tiles + 1
    int n_tiles = 0;
    int tile_G = 1;
    int tile_cfg = 0;            // 7: built for (and launched with) the dense geometry TileCfg7; 0: the hierarchy's default
    // value codes (tile kernels only): at most kMaxCodes distinct values (by bit pattern), entry k's value is
    // dict[codes[k]].  nullptr: fp64 values only.  Ax is kept for every other kernel.
    // pair codes (tile kernels only, in place of value codes): at most kMaxCodes distinct (value, column - row)
    // pairs, entry k of row i is pairs[codes[k]].v at column i + pairs[codes[k]].delta; dict stays nullptr.  Aj and Ax
    // are kept for every other kernel.
    // row codes (one lane per row, in place of the per-entry pair codes, which are then not uploaded: codes stays
    // nullptr): at most kMaxCodes distinct rows, row i's entries are pairs[patterns[rcodes[i]].pair[k]]; the pattern
    // table is padded to kMaxCodes entries, npatterns of them used
    unsigned char *codes = nullptr;
    double *dict = nullptr;
    PairCode *pairs = nullptr;
    int ndict = 0;               // entries of dict or pairs
    unsigned char *rcodes = nullptr;
    RowPattern *patterns = nullptr;
    int npatterns = 0;
};

// The operator arrays of a tile launch
static void tile_operator(TileArgs &a, const DevCsr &M)
{
    a.tiles = M.tiles;
    a.Ap = M.Ap; a.Aj = M.Aj; a.Ax = M.Ax;
    a.pairs = M.pairs; a.ndict = M.ndict;
    if (M.rcodes != nullptr) { a.codes = M.rcodes; a.patterns = M.patterns; }
    else { a.codes = M.codes; a.dict = M.dict; }
}

// Operator bytes a launch streams for nz stored entries: 4 B column + 8 B value; when the launch goes to a coded tile
// kernel, 4 B column + 1 B value code plus the 8-B-per-value table, or 1 B pair code plus the 16-B-per-pair table
static double entry_bytes(const DevCsr &M, long long nz, bool tiled)
{
    if (tiled && M.pairs != nullptr) return 1.0 * (double)nz + (double)sizeof(PairCode) * M.ndict;
    return (tiled && M.codes != nullptr) ? 5.0 * (double)nz + 8.0 * M.ndict : 12.0 * (double)nz;
}

// Operator bytes a launch over `rows` rows, nz stored entries and `ntiles` tiles streams: its entries (entry_bytes)
// plus ptr_bytes of row pointers, or, row-coded, 1 B per row, the tile descriptors and both tables
static double op_bytes(const DevCsr &M, long long rows, long long nz, long long ntiles, bool tiled, double ptr_bytes)
{
    if (tiled && M.rcodes != nullptr)
        return (double)rows + (double)sizeof(TileDesc) * (double)(ntiles + 1) + (double)sizeof(PairCode) * M.ndict +
               (double)sizeof(RowPattern) * M.npatterns;
    return entry_bytes(M, nz, tiled) + ptr_bytes;
}

// Distinct values of Ax by bit pattern (so -0.0 / +0.0 and NaN payloads stay apart), in order of first appearance,
// and each entry's index among them.  False when there are more than kMaxCodes.
static bool value_codes(const std::vector<double> &Ax, std::vector<unsigned char> &codes, std::vector<double> &dict)
{
    constexpr int kSlots = 4 * kMaxCodes;                  // open addressing, at most a quarter full
    uint64_t key[kSlots];
    int idx[kSlots];
    std::fill(idx, idx + kSlots, -1);
    codes.resize(Ax.size());
    dict.clear();
    uint64_t last = 0;
    int last_code = -1;
    for (size_t k = 0; k < Ax.size(); k++) {
        uint64_t u;
        memcpy(&u, &Ax[k], sizeof u);
        if (last_code < 0 || u != last) {
            size_t h = (size_t)((u * 0x9E3779B97F4A7C15ull) >> 54) & (kSlots - 1);
            while (idx[h] >= 0 && key[h] != u) h = (h + 1) & (kSlots - 1);
            if (idx[h] < 0) {
                if ((int)dict.size() == kMaxCodes) return false;
                key[h] = u;
                idx[h] = (int)dict.size();
                dict.push_back(Ax[k]);
            }
            last = u;
            last_code = idx[h];
        }
        codes[k] = (unsigned char)last_code;
    }
    return true;
}

// Distinct (value bit pattern, column - row) pairs of H's entries, in order of first appearance, and each entry's
// index among them.  False when there are more than kMaxCodes.  Rows take part without special cases: the padding
// (column -1) of a zero-start copy gives a different delta on every row, and so do rectangular P / R and the
// irregular coarse levels, so those exceed the limit on their own unless they are tiny.
static bool pair_codes(const HostCsr &H, std::vector<unsigned char> &codes, std::vector<PairCode> &pairs)
{
    constexpr int kSlots = 4 * kMaxCodes;                  // open addressing, at most a quarter full
    uint64_t key_v[kSlots];
    int key_d[kSlots];
    int idx[kSlots];
    std::fill(idx, idx + kSlots, -1);
    codes.resize(H.Aj.size());
    pairs.clear();
    uint64_t last_v = 0;
    int last_d = 0, last_code = -1;
    for (int i = 0; i < H.n_rows; i++) {
        for (int k = H.Ap[(size_t)i]; k < H.Ap[(size_t)i + 1]; k++) {
            uint64_t u;
            memcpy(&u, &H.Ax[(size_t)k], sizeof u);
            const int d = H.Aj[(size_t)k] - i;
            if (last_code < 0 || u != last_v || d != last_d) {
                const uint64_t hk = u ^ ((uint64_t)(uint32_t)d * 0xC2B2AE3D27D4EB4Full);
                size_t h = (size_t)((hk * 0x9E3779B97F4A7C15ull) >> 54) & (kSlots - 1);
                while (idx[h] >= 0 && (key_v[h] != u || key_d[h] != d)) h = (h + 1) & (kSlots - 1);
                if (idx[h] < 0) {
                    if ((int)pairs.size() == kMaxCodes) return false;
                    key_v[h] = u;
                    key_d[h] = d;
                    idx[h] = (int)pairs.size();
                    PairCode p;
                    p.v = H.Ax[(size_t)k];
                    p.delta = d;
                    p.pad_ = 0;
                    pairs.push_back(p);
                }
                last_v = u;
                last_d = d;
                last_code = idx[h];
            }
            codes[(size_t)k] = (unsigned char)last_code;
        }
    }
    return true;
}

// Distinct rows of a pair-coded operator (codes from pair_codes): the sequences of their pair codes, in order of first
// appearance, and each row's index among them.  False when there are more than kMaxCodes or a row is longer than
// kRowCodeMaxLen.
static bool row_codes(const HostCsr &H, const std::vector<unsigned char> &codes, std::vector<unsigned char> &rc,
                      std::vector<RowPattern> &pats)
{
    constexpr int kSlots = 4 * kMaxCodes;                  // open addressing, at most a quarter full
    int idx[kSlots];
    std::fill(idx, idx + kSlots, -1);
    rc.resize((size_t)H.n_rows);
    pats.clear();
    RowPattern last;
    int last_code = -1;
    for (int i = 0; i < H.n_rows; i++) {
        const int k0 = H.Ap[(size_t)i], len = H.Ap[(size_t)i + 1] - k0;
        if (len > kRowCodeMaxLen) return false;
        RowPattern p;
        memset(&p, 0, sizeof p);
        p.len = (unsigned char)len;
        if (len > 0) memcpy(p.pair, &codes[(size_t)k0], (size_t)len);
        if (last_code < 0 || memcmp(&p, &last, sizeof p) != 0) {
            uint64_t w[2];
            memcpy(w, &p, sizeof w);
            const uint64_t hk = w[0] ^ (w[1] * 0xC2B2AE3D27D4EB4Full);
            size_t h = (size_t)((hk * 0x9E3779B97F4A7C15ull) >> 54) & (kSlots - 1);
            while (idx[h] >= 0 && memcmp(&pats[(size_t)idx[h]], &p, sizeof p) != 0) h = (h + 1) & (kSlots - 1);
            if (idx[h] < 0) {
                if ((int)pats.size() == kMaxCodes) return false;
                idx[h] = (int)pats.size();
                pats.push_back(p);
            }
            last = p;
            last_code = idx[h];
        }
        rc[(size_t)i] = (unsigned char)last_code;
    }
    return true;
}

struct WaveSchedule {       // a sequential sweep over a row list, regrouped into dependency waves
    int *rows = nullptr;    // device, wave-major (level numbering)
    std::vector<long long> ptr;   // wave w = rows[ptr[w] .. ptr[w+1])
    std::vector<long long> nnz;   // stored entries of the rows of wave w (roofline accounting)
    bool contiguous = false;      // rows of wave w are exactly ptr[w] .. ptr[w+1]-1 (wave-major permuted level)
    std::vector<int> tile_ptr;    // contiguous: tiles of wave w = [tile_ptr[w], tile_ptr[w+1])
};

// Zero-start copy of a wave-major level operator (build_zero_start): what a forward sweep's first pass needs when it
// starts from x = 0.  Wave w of that pass reads only zeros from the columns of waves >= w, so the copy keeps each
// row's diagonal and its entries in earlier waves, each in the lane that sums it in the full launch.
struct ZeroStart {
    DevCsr A;                        // Ap == nullptr: no copy (the level keeps the full operator)
    std::vector<int> tile_ptr;       // tiles of wave w = [tile_ptr[w], tile_ptr[w+1])
    std::vector<long long> nnz;      // stored entries (padding included) of the rows of wave w
    std::vector<char> tile;          // wave w is laid out for the tile kernel (else for the rows kernel)
};

struct SmootherSpec {       // host copy of an amgb_smoother
    int kind = AMGB_SM_NONE, iterations = 1, sweep = 0, bs = 1;
    double omega = 1.0;
    bool has_list = false;
    std::vector<int> list;
    std::vector<double> Dinv;
    // SURVEY 8(f)-2 smoothers
    std::vector<int> list2;          // CF/FC Jacobi: F-points (list = C-points)
    int f_iterations = 1, c_iterations = 1;
    std::vector<double> coef;        // polynomial, descending order
};

struct Smoother {
    int kind = AMGB_SM_NONE;
    int iterations = 1;
    int sweep = AMGB_SWEEP_FORWARD;
    int bs = 1;
    double omega = 1.0;
    WaveSchedule ws;
    double *Dinv = nullptr;
    // indexed Jacobi sweeps (jacobi_indexed: rows1; CF/FC Jacobi: rows1 = C-points, rows2 = F-points), level numbering
    int *rows1 = nullptr, *rows2 = nullptr;
    long long n_rows1 = 0, n_rows2 = 0;
    int f_iterations = 1, c_iterations = 1;
    bool cf_contig = false;          // CF/FC Jacobi on a level stored C|F: ws.ptr = {0, nC, n} (+ tile ranges)
    // normal-equation smoothers: column-sorted copies of A (ne_A) and A^T (ne_At; omega-scaled for jacobi_ne),
    // inverse diagonal of A A^H or A^H A in Dinv, conflict waves of the sweep operator in ws (row lists)
    DevCsr ne_A, ne_At;
    // Schwarz: subdomain row lists (sz_Sj / sz_Sp), block inverses (Dinv) with offsets sz_Tp, largest subdomain
    int *sz_Sj = nullptr, *sz_Sp = nullptr;
    long long *sz_Tp = nullptr;
    int sz_max_m = 0;
    std::vector<double> coef;        // polynomial coefficients (host: they become kernel arguments)
    // EXPERIMENTAL resident-vector cluster sweep (AMGB_RESIDENT=1): device copies of the schedule
    long long *res_wave_ptr = nullptr;
    int *res_seq = nullptr;
    int res_seq_len = 0, res_log2m = 0, res_csize = 0;
    double res_bytes = 0.0;
};

struct ProfRec {               // one launch of a profiled cycle (amgb_profile_cycle)
    int level, op, lanes;
    long long rows, nnz;
    double bytes;
    cudaEvent_t e0, e1;
};

struct HostLevel {
    HostCsr A, P, R;
    bool has_pr = false;
    SmootherSpec pre, post;
};

struct Level {
    DevCsr A, P, R;
    ZeroStart zs;                    // levels >= 1 whose pre-smoother sweeps forward over the wave-major layout
    bool has_pr = false;
    Smoother pre, post;
    double *x = nullptr, *x_home = nullptr, *xalt = nullptr, *b = nullptr, *r = nullptr;
    double *poly[2] = {nullptr, nullptr};     // polynomial smoother: Horner accumulator h and A h
    // AMLI cycle (allocated on first use): the two search directions, A_c p, the accumulated coarse correction
    // and four device scalars (<p0,b>, <p0,Ap0>, <p1,b> | <p0,Ap1'>, <p1,Ap1>)
    double *amli_p[2] = {nullptr, nullptr}, *amli_Ap = nullptr, *amli_x = nullptr, *amli_s = nullptr;
};

// K-wide level vectors of amgb_solve_many (abi_many.cuh), n x K row-major; one set per width K = 2, 4, 8
struct ManyLevel {
    double *x = nullptr, *x_home = nullptr, *xalt = nullptr, *b = nullptr, *r = nullptr;
    double *poly[2] = {nullptr, nullptr};     // levels with a polynomial smoother: Horner accumulator h and A h
};
struct ManyWidth {
    std::vector<ManyLevel> lv;        // empty until the first batched solve of this width
    double *partials = nullptr;       // K per block of the level-0 residual launch
    double *norms2 = nullptr;         // (cap) x K squared residual norms
    int norms2_cap = 0;
    double *io = nullptr;             // n0 x K: the caller's column slice in its own row order
    // n0 x K Krylov blocks (abi_many_krylov.cuh, on the first batched CG / BiCGStab / GMRES solve of this width):
    // x, p, Ap, b for CG; BiCGStab adds r, r*, s, A M s; GMRES (abi_many_gmres.cuh) takes the first seven
    double *kry[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaGraphExec_t graph[3] = {nullptr, nullptr, nullptr};   // per cycle kind V / W / F
    int graph_cpl[3] = {0, 0, 0};
    long long graph_nodes[3] = {0, 0, 0};
};

static int validate_matrix(const amgb_matrix *M, const char *name)
{
    if (M == nullptr) return fail(AMGB_EINVAL, std::string(name) + ": null matrix");
    if (M->block_r < 1 || M->block_c < 1) return fail(AMGB_EINVAL, std::string(name) + ": bad blocksize");
    if (M->n_rows < 0 || M->n_cols < 0 || M->n_rows % M->block_r || M->n_cols % M->block_c)
        return fail(AMGB_EINVAL, std::string(name) + ": dimensions not divisible by blocksize");
    if (M->indptr == nullptr || (M->nnz_blocks > 0 && (M->indices == nullptr || M->data == nullptr)))
        return fail(AMGB_EINVAL, std::string(name) + ": null arrays");
    const int nb = M->n_rows / M->block_r;
    if (M->indptr[0] != 0 || (long long)M->indptr[nb] != M->nnz_blocks)
        return fail(AMGB_EINVAL, std::string(name) + ": indptr inconsistent with nnz");
    if (M->nnz_blocks * M->block_r * M->block_c > 2147483647LL - 16)
        return fail(AMGB_EINVAL, std::string(name) + ": nnz exceeds int32 (reference index type)");
    return AMGB_OK;
}

// BSR -> point CSR keeping the storage order (block by block, columns ascending inside a block):
// the per-row summation order then equals scipy's bsr_matvec.
static int to_host_csr(const amgb_matrix *M, HostCsr &H, const char *name)
{
    RET(validate_matrix(M, name));
    const int R = M->block_r, C = M->block_c, nb = M->n_rows / R;
    H.n_rows = M->n_rows;
    H.n_cols = M->n_cols;
    const long long nnz = M->nnz_blocks * R * C;
    H.Ap.resize((size_t)M->n_rows + 1);
    H.Aj.resize((size_t)nnz);
    H.Ax.resize((size_t)nnz);
    const int ncb = M->n_cols / C;
    if (R == 1 && C == 1) {
        std::copy(M->indptr, M->indptr + nb + 1, H.Ap.begin());
        std::copy(M->indices, M->indices + nnz, H.Aj.begin());
        std::copy(M->data, M->data + nnz, H.Ax.begin());
        for (long long k = 0; k < nnz; k++)
            if (H.Aj[k] < 0 || H.Aj[k] >= M->n_cols)
                return fail(AMGB_EINVAL, std::string(name) + ": column index out of range");
        for (int i = 0; i < nb; i++)
            if (H.Ap[i + 1] < H.Ap[i]) return fail(AMGB_EINVAL, std::string(name) + ": indptr not monotone");
        return AMGB_OK;
    }
    long long pos = 0;
    for (int I = 0; I < nb; I++) {
        const int s = M->indptr[I], e = M->indptr[I + 1];
        if (e < s) return fail(AMGB_EINVAL, std::string(name) + ": indptr not monotone");
        for (int r = 0; r < R; r++) {
            H.Ap[(size_t)I * R + r] = (int)pos;
            for (int jj = s; jj < e; jj++) {
                const int J = M->indices[jj];
                if (J < 0 || J >= ncb) return fail(AMGB_EINVAL, std::string(name) + ": block column out of range");
                const double *blk = M->data + (size_t)jj * R * C + (size_t)r * C;
                for (int c = 0; c < C; c++) {
                    H.Aj[pos] = J * C + c;
                    H.Ax[pos] = blk[c];
                    pos++;
                }
            }
        }
    }
    H.Ap[M->n_rows] = (int)pos;
    return AMGB_OK;
}

// sequential sweep over `list` (nullptr = 0..n-1) -> dependency waves.  Position k (row i) goes to
// wave 1 + max(last write wave of any j it reads, last wave in which x_i was read or written), so
// executing waves in order, rows of one wave concurrently, reproduces the sequential result.
static void build_waves(const HostCsr &A, const int *list, long long m, std::vector<int> &rows_sorted,
                        std::vector<long long> &ptr)
{
    const int n = A.n_rows;
    std::vector<int> wwave((size_t)n, 0), rwave((size_t)n, 0), w((size_t)m);
    int maxw = 0;
    for (long long k = 0; k < m; k++) {
        const int i = list ? list[k] : (int)k;
        int wv = std::max(rwave[i], wwave[i]);
        for (int jj = A.Ap[i]; jj < A.Ap[i + 1]; jj++) {
            const int j = A.Aj[jj];
            if (j != i && j < n) wv = std::max(wv, wwave[j]);
        }
        wv += 1;
        w[(size_t)k] = wv;
        wwave[i] = wv;
        for (int jj = A.Ap[i]; jj < A.Ap[i + 1]; jj++) {
            const int j = A.Aj[jj];
            if (j != i && j < n) rwave[j] = std::max(rwave[j], wv);
        }
        maxw = std::max(maxw, wv);
    }
    ptr.assign((size_t)maxw + 1, 0);
    for (long long k = 0; k < m; k++) ptr[(size_t)w[(size_t)k]]++;
    for (int q = 0; q < maxw; q++) ptr[(size_t)q + 1] += ptr[(size_t)q];
    rows_sorted.resize((size_t)m);
    std::vector<long long> cur(ptr.begin(), ptr.end() - 1);
    for (long long k = 0; k < m; k++) {
        const int i = list ? list[k] : (int)k;
        rows_sorted[(size_t)cur[(size_t)w[(size_t)k] - 1]++] = i;
    }
    for (int q = 0; q < maxw; q++)   // ascending rows inside a wave: better locality, same result
        std::sort(rows_sorted.begin() + ptr[(size_t)q], rows_sorted.begin() + ptr[(size_t)q + 1]);
}

// B = A[order, :][:, colpos]  (order: new row -> old row, or null; colpos: old col -> new col, or null);
// the entry order inside a row is kept, so per-row summation order is unchanged.
static void permute_csr(const HostCsr &A, const int *order, const int *colpos, HostCsr &B)
{
    B.n_rows = A.n_rows;
    B.n_cols = A.n_cols;
    B.Ap.resize(A.Ap.size());
    B.Aj.resize(A.Aj.size());
    B.Ax.resize(A.Ax.size());
    long long pos = 0;
    for (int i = 0; i < A.n_rows; i++) {
        const int o = order ? order[i] : i;
        B.Ap[(size_t)i] = (int)pos;
        for (int jj = A.Ap[o]; jj < A.Ap[o + 1]; jj++) {
            B.Aj[(size_t)pos] = colpos ? colpos[A.Aj[jj]] : A.Aj[jj];
            B.Ax[(size_t)pos] = A.Ax[jj];
            pos++;
        }
    }
    B.Ap[(size_t)A.n_rows] = (int)pos;
}

// the reference's sweeps let the LAST stored diagonal entry of a row win (relaxation.h:60-66); the flat-gather
// kernel keeps one slot per row and therefore only takes matrices without such duplicates
static bool has_duplicate_diagonal(const HostCsr &A)
{
    for (int i = 0; i < A.n_rows; i++) {
        int cnt = 0;
        for (int jj = A.Ap[(size_t)i]; jj < A.Ap[(size_t)i + 1]; jj++) cnt += (A.Aj[(size_t)jj] == i);
        if (cnt > 1) return true;
    }
    return false;
}

static int pick_tile_G(const Settings &S, long long nnz, long long n_rows)
{
    if (S.tile_G != 0) return S.tile_G;
    if (n_rows <= 0) return 1;
    const double avg = (double)nnz / (double)n_rows;
    int g = 1;
    while (g < 32 && avg > S.lane_entries * g) g <<= 1;     // ~6-12 stored entries per lane (default)
    return g;
}

// whole rows, <= T entries and <= RMAX rows per tile, no tile across a `breaks` row (sorted, e.g. Gauss-Seidel wave
// boundaries); a row longer than T is a tile of its own.
// Row counts are rounded down to a multiple of the rows reduced per pass (32/G) where possible.
static void build_tiles(const HostCsr &A, int G, int T, int rmax, const std::vector<long long> *breaks,
                        std::vector<TileDesc> &tiles, std::vector<int> *tile_ptr)
{
    const int n = A.n_rows, rpp = 32 / G;
    tiles.clear();
    size_t bi = 1;                       // next break to honour: (*breaks)[bi]
    int r = 0;
    while (r < n) {
        long long limit = n;
        if (breaks) {
            while (bi < breaks->size() && (*breaks)[bi] <= r) {
                bi++;
            }
            if (bi < breaks->size()) limit = (*breaks)[bi];
        }
        int e = r;
        long long nz = 0;
        while (e < limit && e - r < rmax) {
            const long long len = A.Ap[(size_t)e + 1] - A.Ap[(size_t)e];
            if (nz + len > T) break;
            nz += len;
            e++;
        }
        if (e == r) {
            e = r + 1;                                   // a single long row
        } else if (e < limit && e - r > rpp) {
            e = r + ((e - r) / rpp) * rpp;               // full passes only
        }
        tiles.push_back(TileDesc{r, A.Ap[(size_t)r]});
        r = e;
    }
    tiles.push_back(TileDesc{n, A.Ap[(size_t)n]});       // sentinel
    if (tile_ptr && breaks) {
        // tile range of every [breaks[w], breaks[w+1]) row range (empty ranges allowed): tiles start on breaks
        tile_ptr->clear();
        size_t t = 0;
        for (size_t w = 0; w < breaks->size(); w++) {
            while (t + 1 < tiles.size() && tiles[t].row0 < (*breaks)[w]) t++;
            tile_ptr->push_back((int)t);
        }
    }
}

// A zero-start copy may replace the full operator only where dropping v * (+0) terms cannot change a sum: every value
// is finite (inf * 0 = NaN), and each row has at most one diagonal entry (the last stored duplicate would win).
static bool zero_start_eligible(const HostCsr &A)
{
    if (A.n_rows != A.n_cols) return false;
    for (double v : A.Ax)
        if (!std::isfinite(v)) return false;
    return !has_duplicate_diagonal(A);
}

// Entries of the zero-start copy (ZeroStart) of a wave-major operator, wave w = rows [wptr[w], wptr[w+1]).
// Lane s of the g lanes that reduce a row takes the row's entries s, s+g, s+2g, ... (csr_rows_kernel and
// csr_tile_kernel alike).  Lane s's k-th kept entry goes to position k g + s; positions a shorter lane leaves open
// hold padding (col -1, +0.0), which the kernels skip.  So every kept term is added in the same lane and order as in
// the full launch, and each dropped term was v * (+0) = +-0, which leaves a partial sum that starts at +0 unchanged:
// the row sums are bit-identical.  The diagonal is never summed, so it goes to the lane with the fewest kept entries.
// tile[w]: wave w runs on the tile kernel (g = G; a row longer than T is reduced by the whole warp, g = 32, and is
// padded past T so that it stays on that path), else on the rows kernel (g = lanes).
static void build_zero_start(const HostCsr &A, const std::vector<long long> &wptr, const std::vector<char> &tile, int G,
                             int lanes, int T, HostCsr &Z, std::vector<long long> &wnnz)
{
    const int n = A.n_rows;
    const size_t nw = wptr.size() - 1;
    std::vector<int> wave_of((size_t)n, (int)nw);        // rows outside the sweep are never written: treat as later
    for (size_t w = 0; w < nw; w++)
        for (long long i = wptr[w]; i < wptr[w + 1]; i++) wave_of[(size_t)i] = (int)w;
    Z = HostCsr();
    Z.n_rows = A.n_rows;
    Z.n_cols = A.n_cols;
    Z.Ap.assign((size_t)n + 1, 0);
    wnnz.assign(nw, 0);
    for (size_t w = 0; w < nw; w++) {
        for (long long i = wptr[w]; i < wptr[w + 1]; i++) {
            const int s0 = A.Ap[(size_t)i], len = A.Ap[(size_t)i + 1] - s0;
            const bool whole_warp = tile[w] && len > T;
            const int g = tile[w] ? (whole_warp ? 32 : G) : lanes;
            auto kept = [&](int c) { return c != i && wave_of[(size_t)c] < (int)w; };
            int cnt[32] = {0};
            int jdiag = -1;
            for (int q = 0; q < len; q++) {
                const int c = A.Aj[(size_t)s0 + q];
                if (c == i) jdiag = s0 + q;
                else if (kept(c)) cnt[q % g]++;
            }
            int dl = 0;                                   // the diagonal's lane
            for (int s = 1; s < g; s++)
                if (cnt[s] < cnt[dl]) dl = s;
            if (jdiag >= 0) cnt[dl]++;
            long long rl = 0;                             // the copy's row length
            for (int s = 0; s < g; s++)
                if (cnt[s] > 0) rl = std::max<long long>(rl, (long long)(cnt[s] - 1) * g + s + 1);
            if (whole_warp) rl = std::max<long long>(rl, (long long)(T / 32 + 1) * 32);
            const size_t base = Z.Aj.size();
            Z.Aj.resize(base + (size_t)rl, -1);
            Z.Ax.resize(base + (size_t)rl, 0.0);
            int k[32] = {0};
            for (int q = 0; q < len; q++) {
                const int c = A.Aj[(size_t)s0 + q];
                if (!kept(c)) continue;
                const int s = q % g;
                const size_t p = base + (size_t)k[s]++ * g + s;
                Z.Aj[p] = c;
                Z.Ax[p] = A.Ax[(size_t)s0 + q];
            }
            if (jdiag >= 0) {
                const size_t p = base + (size_t)k[dl] * g + dl;
                Z.Aj[p] = (int)i;
                Z.Ax[p] = A.Ax[(size_t)jdiag];
            }
            Z.Ap[(size_t)i + 1] = (int)Z.Aj.size();
            wnnz[w] += rl;
        }
    }
}

// A level's row layout as finalize_levels decides it from the level's pattern and smoothers: the wave-major (or C|F)
// permutation, empty = natural numbering, and the contiguous schedule of that layout
struct LevelLayout {
    std::vector<int> order, pos;      // order[new] = old, pos[old] = new
    WaveSchedule W;
    int src = -1;                     // 0 / 1 = waves of pre / post, 2 / 3 = C|F layout of pre / post, -1 = none
};

// How upload_csr streams an operator's values to the tile kernels (the decision lives in value_stream)
struct ValueStream {
    enum { FP64 = 0, VALUE = 1, PAIR = 2, ROW = 3 };
    int format = FP64;
    std::vector<unsigned char> codes;     // VALUE / PAIR: one per entry; ROW: one per row
    std::vector<double> dict;             // VALUE
    std::vector<PairCode> pairs;          // PAIR / ROW
    std::vector<RowPattern> pats;         // ROW
};

// amgb_hierarchy_replace_level0's same-pattern state, built on the first such call: the source pattern level 0 was
// built from, and for the column-sorted copy and its transpose that normal-equation / Schwarz smoothers keep, the
// source entry of every device slot
struct Level0Refresh {
    bool have_pattern = false;
    std::vector<int> Ap, Aj;
    int *map_sorted = nullptr, *map_T = nullptr;
};

// ------------------------------------------------------------------------------------------
// the engine
// ------------------------------------------------------------------------------------------
struct amgb_hierarchy {
    int device = 0;
    Settings S;                       // the launch settings this hierarchy was created under
    std::vector<HostLevel> host;      // until finalize
    std::vector<Level> levels;
    std::vector<void *> allocs;
    long long dev_bytes = 0;
    bool finalized = false;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    // AMGB_FLAG_DEVICE_IO calls: the caller's stream (null = `stream`) and the events ordering the two (CallerIo)
    cudaStream_t io_stream = nullptr;
    cudaEvent_t io_event[2] = {nullptr, nullptr};

    std::vector<double> coarse_host;
    double *coarse_pinv = nullptr;
    int coarse_n = 0;
    bool coarse_zero = false;
    bool have_coarse = false;
    // relaxation as the coarse solver (multilevel.py:764-781): x = 0, then `iterations` sweeps of a smoother
    bool coarse_relax = false;
    SmootherSpec coarse_spec;
    Smoother coarse_sm;

    // level-0 wave-major permutation (device): order0[new] = old, pos0[old] = new; null = identity
    int *order0 = nullptr, *pos0 = nullptr;
    double *io_tmp = nullptr;

    double *partials = nullptr;   // level-0 residual-norm partial sums
    long long n_partials = 0;
    double *norms2 = nullptr;     // device array of squared residual norms
    int norms2_cap = 0;
    double *norm_host = nullptr;  // pinned scalar for the tol test
    double *sumsq_parts = nullptr;
    double *kry[4] = {nullptr, nullptr, nullptr, nullptr};   // Krylov work vectors (allocated on first use)
    double *kry2[4] = {nullptr, nullptr, nullptr, nullptr};  // BiCGStab's additional four
    // A^H of level 0 in level-0 numbering (amgb_hierarchy_set_transpose0): CGNR / CGNE only, uploaded on their first
    // call; Ap == nullptr until then
    DevCsr At0;
    // Householder GMRES / FGMRES (amgb_solve_gmres): reflectors W, preconditioned directions Z (flexible), work
    // vectors in the original numbering (v, x, b, update) and in level-0 numbering (b, SpMV in/out), device scalars
    double *gm_W = nullptr, *gm_Z = nullptr, *gm_vec[4] = {nullptr, nullptr, nullptr, nullptr};
    double *gm_lvl[3] = {nullptr, nullptr, nullptr}, *gm_s = nullptr;
    int gm_inner = 0;
    bool gm_flex = false;
    // batched GMRES / FGMRES (amgb_solve_many_gmres): one reflector store for the largest shape asked so far,
    // (max_inner + 1) x npad x K doubles of W, plus max_inner x npad x K of Z when flexible (abi_many_gmres.cuh)
    double *mgm_store = nullptr;
    long long mgm_count = 0;
    // modified Gram-Schmidt GMRES (AMGB_FLAG_MGS, single and batched): device H-column coefficients and ||v||^2
    // partials, grown to the largest shape asked so far (gmres_mgs_scratch in abi_krylov.cuh)
    double *gm_mgs = nullptr;
    long long gm_mgs_count = 0;

    ManyWidth many[3];                // amgb_solve_many, K = 2, 4, 8

    // level 0's smoother descriptors as last uploaded, without Dinv (amgb_hierarchy_replace_level0 compares them)
    SmootherSpec spec0[2];
    Level0Refresh re0;
    std::unordered_map<void *, long long> alloc_bytes;   // size of every live dalloc block (release)

    cudaGraphExec_t graph[4] = {nullptr, nullptr, nullptr, nullptr};
    int graph_cpl[4] = {0, 0, 0, 0};
    long long graph_nodes[4] = {0, 0, 0, 0};
    bool profiling = false;
    int cur_level = 0;
    std::vector<ProfRec> prof;
    long long launches = 0;        // kernels issued by the current (or captured) sequence
    long long last_launches = 0;

    // coarse tail: levels >= tail_level run inside one cluster kernel (tail_kernel.cuh), or in grid mode
    // (S.tail_grid, grid_kernel.cuh) the same recorded program walked by one cooperatively launched CTA per SM
    int tail_level = 1 << 30;
    int tail_csize = 1;
    GridSync *grid_sync = nullptr;
    bool fuse_stop = false;        // issuing the cycle whose level-0 post-smoother also computes the stop test's residual
    long long stop_nparts = 0;     // partials that cycle writes
    cudaGraphExec_t graph_stop[4] = {nullptr, nullptr, nullptr, nullptr};
    int graph_stop_cpl[4] = {0, 0, 0, 0};
    long long graph_stop_nodes[4] = {0, 0, 0, 0};
    bool recording = false;
    std::vector<TailStep> rec;
    double rec_bytes = 0.0;
    struct TailProg { TailStep *dev = nullptr; int n = 0, cpl = -1, lvl = -1; double bytes = 0.0; } tail_prog[4];

    int record(int op, int G, int row0, int nrows, const int *rows, const DevCsr *M, const double *x,
               const double *b, double *y, double omega, double bytes, const double *dense = nullptr, int ncols = 0)
    {
        TailStep st;
        // small steps run on CTA 0 alone (no cluster barrier); the bound is on the bytes one SM must pull
        const int nctas = S.tail_grid ? S.grid_ctas : tail_csize;
        const bool solo = nctas > 1 && bytes <= S.tail_solo_bytes;
        if (op <= T_GS && nrows > 0) {
            // one pass over the step's rows: as many lanes per row as the cluster can spare, but no more
            // than the row length warrants (G from pick_lanes is the smallest power of two >= mean length)
            const int nthreads = (solo ? 1 : nctas) * kTailThreads;
            int fill = 1;
            while (fill < 32 && (long long)fill * 2 * nrows <= nthreads) fill <<= 1;
            G = std::max(1, std::min(G, fill));
        }
        st.op = op; st.G = G; st.row0 = row0; st.nrows = nrows; st.rows = rows;
        st.Ap = M ? M->Ap : nullptr; st.Aj = M ? M->Aj : nullptr; st.Ax = M ? M->Ax : dense;
        st.x = x; st.b = b; st.y = y; st.omega = omega; st.ncols = ncols; st.solo = solo ? 1 : 0;
        rec.push_back(st);
        rec_bytes += bytes;
        return AMGB_OK;
    }

    template <typename T>
    int dalloc(T **p, long long count)
    {
        *p = nullptr;
        size_t bytes = (size_t)std::max<long long>(count, 1) * sizeof(T);
        bytes = (bytes + 255) & ~(size_t)255;
        void *q = nullptr;
        CK(cudaMalloc(&q, bytes));
        allocs.push_back(q);
        alloc_bytes[q] = (long long)bytes;
        dev_bytes += (long long)bytes;
        *p = (T *)q;
        return AMGB_OK;
    }

    // dfree that also takes the block out of dev_bytes (level-0 replacement frees what it rebuilds)
    template <typename T>
    void release(T *&p)
    {
        if (p == nullptr) return;
        auto it = alloc_bytes.find((void *)p);
        if (it != alloc_bytes.end()) { dev_bytes -= it->second; alloc_bytes.erase(it); }
        dfree(p);
    }
    void release_csr(DevCsr &D)
    {
        release(D.Ap); release(D.Aj); release(D.Ax); release(D.tiles);
        release(D.codes); release(D.dict); release(D.pairs); release(D.rcodes); release(D.patterns);
        D = DevCsr();
    }

    // give a buffer of this pool back before the hierarchy dies (re-sized Krylov work space)
    template <typename T>
    void dfree(T *&p)
    {
        if (p == nullptr) return;
        auto it = std::find(allocs.begin(), allocs.end(), (void *)p);
        if (it != allocs.end()) allocs.erase(it);
        cudaFree((void *)p);
        p = nullptr;
    }

    // `pad` extra elements are allocated (and zeroed) past the payload: the TMA reads whole 16-byte groups
    template <typename T>
    int upload(T **p, const T *src, long long count, int pad = 0)
    {
        RET(dalloc(p, count + pad));
        if (pad > 0) CK(cudaMemset((void *)(*p + count), 0, sizeof(T) * (size_t)pad));
        if (count > 0) CK(cudaMemcpy(*p, src, (size_t)count * sizeof(T), cudaMemcpyHostToDevice));
        return AMGB_OK;
    }

    // role: 0 = a level operator A, 1 = prolongation P, 2 = restriction R (flat-gather mode 2 picks by it)
    // like: launch geometry (lanes, tile G, tile configuration) to keep instead of choosing it from H's row lengths
    // code_values: also upload pair codes when the operator has at most kMaxCodes distinct (value, column - row) pairs
    // and a pair-coded kernel exists for its launch geometry (default or dense tiles, G <= kPairMaxG, no programmatic
    // launch), else value codes when it has at most kMaxCodes distinct values and its tile geometry has coded kernels
    // (the default and the dense one)
    int upload_csr(const HostCsr &H, DevCsr &D, const std::vector<long long> *breaks = nullptr,
                   std::vector<int> *tile_ptr = nullptr, int role = 0, int level = 0, const DevCsr *like = nullptr,
                   bool code_values = false)
    {
        D.n_rows = H.n_rows;
        D.n_cols = H.n_cols;
        D.nnz = (long long)H.Aj.size();
        RET(upload(&D.Ap, H.Ap.data(), (long long)H.Ap.size(), 8));
        RET(upload(&D.Aj, H.Aj.data(), D.nnz, 16));       // 16: the coded tile kernels copy 16-entry groups
        RET(upload(&D.Ax, H.Ax.data(), D.nnz, 8));
        D.lanes = like ? like->lanes : pick_lanes(S, D.nnz, D.n_rows);
        if (S.use_tiles) {
            D.tile_G = pick_tile_G(S, D.nnz, D.n_rows);
            const bool flat_here = S.tile_flat == 1 || (S.tile_flat == 2 && (role == 2 || (role == 1 && level >= 1)));
            if (flat_here && !has_duplicate_diagonal(H)) D.tile_G = 0;      // 0 = flat-gather kernel
            const double avg = D.n_rows > 0 ? (double)D.nnz / (double)D.n_rows : 0.0;
            D.tile_cfg = (S.dense_cfg == 7 && D.tile_G != 0 && avg > S.dense_avg) ? 7 : 0;
            if (like) { D.tile_G = like->tile_G; D.tile_cfg = like->tile_cfg; }
            std::vector<TileDesc> tiles;
            build_tiles(H, D.tile_G ? D.tile_G : 32, D.tile_cfg == 7 ? S.dense_T : S.tile_T,   // flat: no row-count rounding
                        D.tile_cfg == 7 ? S.dense_rmax : S.tile_rmax, breaks, tiles, tile_ptr);
            D.n_tiles = (int)tiles.size() - 1;
            RET(upload(&D.tiles, tiles.data(), (long long)tiles.size()));
            ValueStream v;
            value_stream(H, D, code_values, v);
            switch (v.format) {
            case ValueStream::ROW:
                RET(upload(&D.rcodes, v.codes.data(), (long long)D.n_rows, 16));
                D.npatterns = (int)v.pats.size();
                v.pats.resize((size_t)kMaxCodes, RowPattern{});       // the kernel copies the whole table
                RET(upload(&D.patterns, v.pats.data(), (long long)v.pats.size()));
                RET(upload(&D.pairs, v.pairs.data(), (long long)v.pairs.size()));
                D.ndict = (int)v.pairs.size();
                break;
            case ValueStream::PAIR:
                RET(upload(&D.codes, v.codes.data(), D.nnz, 16));
                RET(upload(&D.pairs, v.pairs.data(), (long long)v.pairs.size()));
                D.ndict = (int)v.pairs.size();
                break;
            case ValueStream::VALUE:
                RET(upload(&D.codes, v.codes.data(), D.nnz, 16));
                RET(upload(&D.dict, v.dict.data(), (long long)v.dict.size()));
                D.ndict = (int)v.dict.size();
                break;
            }
        }
        return AMGB_OK;
    }

    // The value stream upload_csr picks for H under D's launch geometry (tile_G, tile_cfg, nnz already set), with
    // its tables and codes
    void value_stream(const HostCsr &H, const DevCsr &D, bool code_values, ValueStream &v) const
    {
        v = ValueStream();
        const bool coded_cfg = code_values && (D.tile_cfg == 7 || S.tile_cfg == 6);
        if (coded_cfg && S.use_pair_codes && D.nnz >= S.pair_min_nnz && D.tile_G != 0 && D.tile_G <= kPairMaxG &&
            !S.tile_pdl && pair_codes(H, v.codes, v.pairs)) {
            // row codes: one lane per row, so every tile launch of the operator goes to csr_rowcode_kernel and
            // the per-entry codes are not needed on the device
            std::vector<unsigned char> rc;
            if (S.use_row_codes && D.tile_G == 1 && D.nnz >= S.row_min_nnz && row_codes(H, v.codes, rc, v.pats)) {
                v.codes.swap(rc);
                v.format = ValueStream::ROW;
            } else {
                v.format = ValueStream::PAIR;
            }
        } else if (coded_cfg && value_codes(H.Ax, v.codes, v.dict)) {
            v.pairs.clear();
            v.format = ValueStream::VALUE;
        }
    }

    // ---- per-launch timing (profile mode only; never inside a graph capture) ----
    // AMGB_NCU_SELECT="level:op:count,...": the next `count` launches of (level, op) of an UN-GRAPHED cycle are
    // bracketed by cudaProfilerStart/Stop, so `ncu --profile-from-start off` captures exactly the launches asked
    // for (one per kernel family and level) instead of the ~1000 launches of a cycle.  Profiling aid only.
    bool ncu_open = false;
    void ncu_gate_begin(int op)
    {
#ifndef AMGB_EMU
        if (S.ncu_select.empty() || recording) return;
        for (auto &sel : S.ncu_select)
            if (sel[0] == cur_level && sel[1] == op && sel[2] > 0) {
                sel[2]--;
                cudaStreamSynchronize(stream);
                cudaProfilerStart();
                ncu_open = true;
                return;
            }
#else
        (void)op;
#endif
    }
    void ncu_gate_end()
    {
#ifndef AMGB_EMU
        if (ncu_open) {
            cudaStreamSynchronize(stream);
            cudaProfilerStop();
            ncu_open = false;
        }
#endif
    }

    int prof_begin(int op, int lanes, long long rows, long long nnz, double bytes)
    {
        if (S.use_graph == false) ncu_gate_begin(op);
        if (!profiling) return AMGB_OK;
        ProfRec r;
        r.level = cur_level; r.op = op; r.lanes = lanes; r.rows = rows; r.nnz = nnz; r.bytes = bytes;
        CK(cudaEventCreate(&r.e0));
        CK(cudaEventCreate(&r.e1));
        CK(cudaEventRecord(r.e0, stream));
        prof.push_back(r);
        return AMGB_OK;
    }
    int prof_end()
    {
        ncu_gate_end();
        if (!profiling) return AMGB_OK;
        CK(cudaEventRecord(prof.back().e1, stream));
        return AMGB_OK;
    }

    // ---- launch sequence pieces (all on `stream`) ----
    int spmv(int op, const DevCsr &M, const double *x, const double *b, double *y, double omega = 0.0,
             double *r = nullptr, double *parts = nullptr)
    {
        if (M.n_rows <= 0) return AMGB_OK;
        // algorithmic bytes (SURVEY.md 8(d)): 12 nnz + 4 (n+1) + 8 per vector pass
        const double vec = (op == OP_SPMV) ? 8.0 * M.n_cols + 8.0 * M.n_rows
                         : (op == OP_PADD) ? 8.0 * M.n_cols + 16.0 * M.n_rows
                         : (op == OP_RESID) ? 24.0 * M.n_rows
                         : (24.0 + (r ? 8.0 : 0.0)) * M.n_rows;
        if (recording)   // same op codes in TailOp for the five CSR epilogues
            return record(op, M.lanes, 0, M.n_rows, nullptr, &M, x, b, y, omega, 12.0 * M.nnz + 4.0 * (M.n_rows + 1) + vec);
        launches++;
        const bool tiled = M.tiles != nullptr && (M.nnz >= S.tile_min_nnz || parts != nullptr);
        RET(prof_begin(op, M.tiles ? M.tile_G : M.lanes, M.n_rows, M.nnz,
                       op_bytes(M, M.n_rows, M.nnz, M.n_tiles, tiled, 4.0 * (M.n_rows + 1)) + vec));
        if (tiled) {
            TileArgs a;
            tile_operator(a, M);
            a.tile_begin = 0; a.tile_end = M.n_tiles;
            a.x = x; a.b = b; a.y = y; a.r = r; a.omega = omega;
            a.partials = parts;
            const int grid = parts ? tile_grid(S, op, 1 << 30, M.tile_cfg) : tile_grid(S, op, M.n_tiles, M.tile_cfg);   // fixed grid when reducing
            RET(launch_tile(S, op, M.tile_G, a, grid, stream, M.tile_cfg));
        } else {
            CsrRowArgs a;
            a.n = M.n_rows; a.row0 = 0; a.rows = nullptr;
            a.Ap = M.Ap; a.Aj = M.Aj; a.Ax = M.Ax;
            a.x = x; a.b = b; a.y = y; a.r = r; a.omega = omega; a.partials = parts;
            RET(launch_csr(S, op, M.lanes, a, stream));
        }
        return prof_end();
    }

    long long partials_used(const DevCsr &M, int op) const   // slots the kernel of `op` actually writes
    {
        return M.tiles ? (long long)S.num_sms * (M.tile_cfg == 7 ? S.dense_ctas[op] : S.tile_ctas[op]) : csr_grid(M.n_rows, M.lanes);
    }
    long long partials_len(const DevCsr &M) const
    {
        // residual / Jacobi / last-wave Gauss-Seidel partial sums: one slot per CTA of the (fixed) persistent grid
        return M.tiles ? (long long)S.num_sms * std::max({S.tile_ctas[OP_RESID], S.tile_ctas[OP_JACOBI], S.tile_ctas[OP_GS],
                                                          S.dense_ctas[OP_RESID], S.dense_ctas[OP_JACOBI], S.dense_ctas[OP_GS]})
                       : csr_grid(M.n_rows, M.lanes);
    }

    // r != nullptr (tile path only, see wave_resid_ok): the wave is the last of its sweep and also writes the residual
    // of its rows to r, their |r|^2 to one partial per CTA of a fixed grid (parts, may be null)
    // zs (r == nullptr only): x holds +0 in every row of waves >= w, so the wave runs on the level's zero-start copy,
    // with the same kernel and lanes as on the full operator (profiled as op 13)
    int gs_wave(const DevCsr &A, const WaveSchedule &ws, long long w, double *x, const double *b, double omega,
                double *r = nullptr, double *parts = nullptr, const ZeroStart *zs = nullptr)
    {
        const int nrow = (int)(ws.ptr[(size_t)w + 1] - ws.ptr[(size_t)w]);
        if (nrow <= 0) return AMGB_OK;
        if (recording)
            return record(T_GS, A.lanes, ws.contiguous ? (int)ws.ptr[(size_t)w] : 0, nrow,
                          ws.contiguous ? nullptr : ws.rows + ws.ptr[(size_t)w], &A, x, b, x, omega,
                          12.0 * ws.nnz[(size_t)w] + 36.0 * nrow);
        launches++;
        const DevCsr &M = zs ? zs->A : A;
        const long long nz = zs ? zs->nnz[(size_t)w] : ws.nnz[(size_t)w];
        const std::vector<int> &tile_ptr = zs ? zs->tile_ptr : ws.tile_ptr;
        // one wave of a sweep: its share of 12 nnz + 4 (n+1) + 4 n (row list) + 24 n
        const bool tiled = r != nullptr || (ws.contiguous && A.tiles != nullptr && ws.nnz[(size_t)w] >= S.tile_min_nnz);
        const long long ntiles = tiled ? tile_ptr[(size_t)w + 1] - tile_ptr[(size_t)w] : 0;
        RET(prof_begin(r ? 12 : zs ? 13 : OP_GS, (ws.contiguous && A.tiles) ? A.tile_G : A.lanes, nrow, nz,
                       op_bytes(M, nrow, nz, ntiles, tiled, 4.0 * nrow) + (r ? 40.0 : 32.0) * nrow));
        if (tiled) {
            TileArgs a;
            tile_operator(a, M);
            a.tile_begin = tile_ptr[(size_t)w]; a.tile_end = tile_ptr[(size_t)w + 1];
            a.x = x; a.b = b; a.y = x; a.r = r; a.omega = omega;
            a.partials = parts;
            const int grid = parts ? tile_grid(S, OP_GS, 1 << 30, M.tile_cfg) : tile_grid(S, OP_GS, a.tile_end - a.tile_begin, M.tile_cfg);
            RET(launch_tile(S, OP_GS, M.tile_G, a, grid, stream, M.tile_cfg));
        } else {
            CsrRowArgs a;
            a.n = nrow;
            a.row0 = ws.contiguous ? (int)ws.ptr[(size_t)w] : 0;
            a.rows = ws.contiguous ? nullptr : ws.rows + ws.ptr[(size_t)w];
            a.Ap = M.Ap; a.Aj = M.Aj; a.Ax = M.Ax;
            a.x = x; a.b = b; a.y = x; a.r = nullptr; a.omega = omega; a.partials = nullptr;
            RET(launch_csr(S, OP_GS, A.lanes, a, stream));
        }
        return prof_end();
    }

    int block_jacobi(Level &L, const Smoother &s);   // defined below (needs its kernel)

    // The wave a Gauss-Seidel smoother runs last, when that launch can also write the residual of its rows
    // (gs_wave with r): the level is stored wave-major and both that wave and the residual run on the tile kernel,
    // whose per-row sums the fused epilogue reproduces.  -1 otherwise.
    long long resid_wave(const Level &L, const Smoother &s, bool with_parts) const
    {
        if (!S.use_wave_resid || recording || s.kind != AMGB_SM_GAUSS_SEIDEL || s.res_seq != nullptr) return -1;
        if (!s.ws.contiguous || s.ws.tile_ptr.empty() || L.A.tiles == nullptr || L.A.tile_G == 0) return -1;
        if (!with_parts && L.A.nnz < S.tile_min_nnz) return -1;
        const long long nw = (long long)s.ws.ptr.size() - 1;
        if (nw < 1 || s.iterations < 1) return -1;
        const long long w = (s.sweep == AMGB_SWEEP_FORWARD) ? nw - 1 : 0;
        return s.ws.nnz[(size_t)w] >= S.tile_min_nnz ? w : -1;
    }

    // smoother, then r = b - A x on the level (multilevel.py:610-612).  parts: |r|^2 partials (null = none); *nparts =
    // how many slots were written.  Where resid_wave allows, the smoother's last wave writes its rows' residual and
    // one launch per remaining contiguous row range completes it.
    int smooth_residual(Level &L, const Smoother &s, double *parts, long long *nparts, bool from_zero = false)
    {
        const long long lw = resid_wave(L, s, parts != nullptr);
        if (lw < 0) {
            RET(smooth(L, s, nullptr, nullptr, from_zero));
            RET(spmv(OP_RESID, L.A, L.x, L.b, L.r, 0.0, nullptr, parts));
            if (nparts) *nparts = partials_used(L.A, OP_RESID);
            return AMGB_OK;
        }
        RET(smooth(L, s, L.r, parts, from_zero));
        long long used = parts ? partials_used(L.A, OP_GS) : 0;
        const long long nw = (long long)s.ws.ptr.size() - 1;
        const long long ranges[2][2] = {{0, lw}, {lw + 1, nw}};
        for (const auto &rg : ranges) {
            if (s.ws.ptr[(size_t)rg[1]] <= s.ws.ptr[(size_t)rg[0]]) continue;
            RET(resid_waves(L, s.ws, rg[0], rg[1], parts ? parts + used : nullptr));
            if (parts) used += partials_used(L.A, OP_RESID);
        }
        if (nparts) *nparts = used;
        return AMGB_OK;
    }

    // the residual of the rows of waves [w0, w1) of a wave-major level (tile kernel)
    int resid_waves(Level &L, const WaveSchedule &ws, long long w0, long long w1, double *parts)
    {
        const DevCsr &M = L.A;
        const long long rows = ws.ptr[(size_t)w1] - ws.ptr[(size_t)w0];
        long long nz = 0;
        for (long long w = w0; w < w1; w++) nz += ws.nnz[(size_t)w];
        launches++;
        const int t0 = ws.tile_ptr[(size_t)w0], t1 = ws.tile_ptr[(size_t)w1];
        RET(prof_begin(OP_RESID, M.tile_G, rows, nz,
                       op_bytes(M, rows, nz, t1 - t0, true, 4.0 * (rows + 1)) + 24.0 * rows));
        TileArgs a;
        tile_operator(a, M);
        a.tile_begin = t0; a.tile_end = t1;
        a.x = L.x; a.b = L.b; a.y = L.r; a.r = nullptr; a.omega = 0.0;
        a.partials = parts;
        const int grid = parts ? tile_grid(S, OP_RESID, 1 << 30, M.tile_cfg) : tile_grid(S, OP_RESID, t1 - t0, M.tile_cfg);
        RET(launch_tile(S, OP_RESID, M.tile_G, a, grid, stream, M.tile_cfg));
        return prof_end();
    }

    // from_zero: x is +0 on entry (descend's fill), so the first forward pass may run on the zero-start copy
    int smooth(Level &L, const Smoother &s, double *r_last = nullptr, double *parts = nullptr, bool from_zero = false)
    {
        switch (s.kind) {
        case AMGB_SM_NONE: return AMGB_OK;
        case AMGB_SM_JACOBI:
            for (int it = 0; it < s.iterations; it++) {
                RET(spmv(OP_JACOBI, L.A, L.x, L.b, L.xalt, s.omega));
                std::swap(L.x, L.xalt);
            }
            return AMGB_OK;
        case AMGB_SM_GAUSS_SEIDEL: {
            if (s.res_seq != nullptr && !recording) return resident_apply(L, s);
            const long long nw = (long long)s.ws.ptr.size() - 1;
            // relaxation.py:326-330: the symmetric sweep recurses WITHOUT omega (plain GS)
            const double om = (s.sweep == AMGB_SWEEP_SYMMETRIC) ? 1.0 : s.omega;
            // r_last: the last launch of the application also writes the residual of its rows (smooth_residual)
            const bool sym1 = s.sweep == AMGB_SWEEP_SYMMETRIC && nw == 1;   // its only launch is the forward one
            // a wave that also writes the residual reads every entry: it keeps the full operator
            const ZeroStart *zs = (from_zero && !recording && s.ws.contiguous && L.zs.A.Ap != nullptr) ? &L.zs : nullptr;
            for (int it = 0; it < s.iterations; it++) {
                const bool fin = it == s.iterations - 1;
                if (s.sweep == AMGB_SWEEP_FORWARD || s.sweep == AMGB_SWEEP_SYMMETRIC)
                    for (long long w = 0; w < nw; w++) {
                        const bool rl = fin && w == nw - 1 && (s.sweep == AMGB_SWEEP_FORWARD || sym1);
                        double *rw = rl ? r_last : nullptr;
                        RET(gs_wave(L.A, s.ws, w, L.x, L.b, om, rw, rl ? parts : nullptr,
                                    (it == 0 && rw == nullptr) ? zs : nullptr));
                    }
                if (s.sweep == AMGB_SWEEP_BACKWARD)
                    for (long long w = nw - 1; w >= 0; w--) {
                        const bool rl = fin && w == 0;
                        RET(gs_wave(L.A, s.ws, w, L.x, L.b, om, rl ? r_last : nullptr, rl ? parts : nullptr));
                    }
                // symmetric: the backward pass starts with the wave the forward pass ended on;
                // relaxing an independent set twice in a row is idempotent (same inputs, same
                // arithmetic), so that launch is skipped -- bit-identical to running it.
                if (s.sweep == AMGB_SWEEP_SYMMETRIC)
                    for (long long w = nw - 2; w >= 0; w--) {
                        const bool rl = fin && w == 0;
                        RET(gs_wave(L.A, s.ws, w, L.x, L.b, om, rl ? r_last : nullptr, rl ? parts : nullptr));
                    }
            }
            return AMGB_OK;
        }
        case AMGB_SM_BLOCK_JACOBI: return block_jacobi(L, s);
        case AMGB_SM_POLYNOMIAL: return polynomial(L, s);
        case AMGB_SM_JACOBI_INDEXED:                                   // relaxation.py:1133-1138
            for (int it = 0; it < s.iterations; it++) RET(jacobi_indexed(L, s.rows1, s.n_rows1, s.omega));
            return AMGB_OK;
        case AMGB_SM_CF_JACOBI:                                        // relaxation.py:1184-1189
        case AMGB_SM_FC_JACOBI:                                        // relaxation.py:1249-1254
            for (int it = 0; it < s.iterations; it++) {
                if (s.kind == AMGB_SM_FC_JACOBI)
                    for (int f = 0; f < s.f_iterations; f++) RET(cf_sweep(L, s, 1));
                for (int c = 0; c < s.c_iterations; c++) RET(cf_sweep(L, s, 0));
                if (s.kind == AMGB_SM_CF_JACOBI)
                    for (int f = 0; f < s.f_iterations; f++) RET(cf_sweep(L, s, 1));
            }
            return AMGB_OK;
        case AMGB_SM_BLOCK_GAUSS_SEIDEL: return block_gauss_seidel(L, s);
        case AMGB_SM_JACOBI_NE:
        case AMGB_SM_GAUSS_SEIDEL_NE:
        case AMGB_SM_GAUSS_SEIDEL_NR: return normal_equations(L, s);
        case AMGB_SM_SCHWARZ: return schwarz(L, s);
        case AMGB_SM_CF_BLOCK_JACOBI:                                  // relaxation.py:1328-1339
        case AMGB_SM_FC_BLOCK_JACOBI:                                  // relaxation.py:1401-1412
            for (int it = 0; it < s.iterations; it++) {
                if (s.kind == AMGB_SM_FC_BLOCK_JACOBI)
                    for (int f = 0; f < s.f_iterations; f++) RET(block_jacobi_indexed(L, s, s.rows2, s.n_rows2));
                for (int c = 0; c < s.c_iterations; c++) RET(block_jacobi_indexed(L, s, s.rows1, s.n_rows1));
                if (s.kind == AMGB_SM_CF_BLOCK_JACOBI)
                    for (int f = 0; f < s.f_iterations; f++) RET(block_jacobi_indexed(L, s, s.rows2, s.n_rows2));
            }
            return AMGB_OK;
        }
        return fail(AMGB_ENOTIMPL, "smoother kind");
    }

    // one Jacobi sweep over the C-points (which = 0) or the F-points (1) of a CF / FC Jacobi smoother
    int cf_sweep(Level &L, const Smoother &s, int which)
    {
        if (!s.cf_contig)
            return which == 0 ? jacobi_indexed(L, s.rows1, s.n_rows1, s.omega) : jacobi_indexed(L, s.rows2, s.n_rows2, s.omega);
        // C|F layout: the set is the contiguous row range [ptr[which], ptr[which+1]).  The sweep reads the iterate
        // in place and writes the range's new values to the spare buffer (rows of the range read each other's OLD
        // values, relaxation.h:394-399), then only that range is copied back -- no snapshot of the whole vector.
        if (recording) return fail(AMGB_ESTATE, "CF Jacobi inside the cluster tail");
        const long long r0 = s.ws.ptr[(size_t)which], nrow = s.ws.ptr[(size_t)which + 1] - r0;
        if (nrow <= 0) return AMGB_OK;
        double *temp = (L.x == L.x_home) ? L.xalt : L.x_home;
        const long long nnzw = s.ws.nnz[(size_t)which];
        launches++;
        const bool tiled = L.A.tiles != nullptr && !s.ws.tile_ptr.empty() && nnzw >= S.tile_min_nnz;
        const long long ntiles = tiled ? s.ws.tile_ptr[(size_t)which + 1] - s.ws.tile_ptr[(size_t)which] : 0;
        RET(prof_begin(8, L.A.tiles ? L.A.tile_G : L.A.lanes, nrow, nnzw,
                       op_bytes(L.A, nrow, nnzw, ntiles, tiled, 4.0 * (nrow + 1)) + 40.0 * nrow));
        if (tiled) {
            TileArgs a;
            tile_operator(a, L.A);
            a.tile_begin = s.ws.tile_ptr[(size_t)which]; a.tile_end = s.ws.tile_ptr[(size_t)which + 1];
            a.x = L.x; a.b = L.b; a.y = temp; a.r = nullptr; a.omega = s.omega;
            a.partials = nullptr;
            RET(launch_tile(S, OP_JACOBI, L.A.tile_G, a, tile_grid(S, OP_JACOBI, a.tile_end - a.tile_begin, L.A.tile_cfg), stream, L.A.tile_cfg));
        } else {
            CsrRowArgs a;
            a.n = (int)nrow; a.row0 = (int)r0; a.rows = nullptr;
            a.Ap = L.A.Ap; a.Aj = L.A.Aj; a.Ax = L.A.Ax;
            a.x = L.x; a.b = L.b; a.y = temp; a.r = nullptr; a.omega = s.omega; a.partials = nullptr;
            RET(launch_csr(S, OP_JACOBI, L.A.lanes, a, stream));
        }
        RET(prof_end());
        CK(cudaMemcpyAsync(L.x + r0, temp + r0, sizeof(double) * (size_t)nrow, cudaMemcpyDeviceToDevice, stream));
        launches++;
        return AMGB_OK;
    }

    // amg_core.jacobi_indexed (relaxation.h:382-427): temp = x, then the listed rows are relaxed from temp.
    // The level's spare iterate buffer is temp; the rows kernel reads it and writes x (rows outside the list
    // keep their values; a zero diagonal rewrites the old value).
    int jacobi_indexed(Level &L, const int *rows, long long m, double omega)
    {
        if (recording) return fail(AMGB_ESTATE, "indexed Jacobi inside the cluster tail");
        if (m <= 0) return AMGB_OK;
        double *temp = (L.x == L.x_home) ? L.xalt : L.x_home;
        RET(copy_vec(temp, L.x, L.A.n_rows));
        launches++;
        // bytes: the listed rows' entries are not known per list here; account the vector traffic + row list
        RET(prof_begin(8, L.A.lanes, m, 0, 16.0 * L.A.n_rows + 28.0 * (double)m));
        CsrRowArgs a;
        a.n = (int)m; a.row0 = 0; a.rows = rows;
        a.Ap = L.A.Ap; a.Aj = L.A.Aj; a.Ax = L.A.Ax;
        a.x = temp; a.b = L.b; a.y = L.x; a.r = nullptr; a.omega = omega; a.partials = nullptr;
        RET(launch_csr(S, OP_JACOBI, L.A.lanes, a, stream));
        return prof_end();
    }

    // relaxation.polynomial (relaxation.py:646-659): per iteration r = b - A x, h = c_0 r,
    // h = c_k r + A h (Horner), x += h.  L.r is free during smoothing (the cycle recomputes it afterwards).
    int polynomial(Level &L, const Smoother &s)
    {
        if (recording) return fail(AMGB_ESTATE, "polynomial smoother inside the cluster tail");
        if (s.coef.empty() || L.poly[0] == nullptr) return fail(AMGB_ESTATE, "polynomial smoother not prepared");
        const long long n = L.A.n_rows;
        for (int it = 0; it < s.iterations; it++) {
            RET(spmv(OP_RESID, L.A, L.x, L.b, L.r));
            double *h = L.poly[0], *Ah = L.poly[1];
            RET(scale_to(h, s.coef[0], L.r, n));
            for (size_t k = 1; k < s.coef.size(); k++) {
                RET(spmv(OP_SPMV, L.A, h, nullptr, Ah));
                RET(axpby(s.coef[k], L.r, 1.0, Ah, n));      // A h + c_k r
                std::swap(h, Ah);
            }
            RET(axpby(1.0, h, 1.0, L.x, n));
        }
        return AMGB_OK;
    }
    int axpby(double a, const double *x, double b, double *y, long long n)
    {
        if (n <= 0) return AMGB_OK;
        axpby_kernel<<<vec_grid(S, n), 256, 0, stream>>>(a, x, b, y, n);
        CK(cudaGetLastError());
        launches++;
        return AMGB_OK;
    }
    int scale_to(double *y, double a, const double *x, long long n)
    {
        if (n <= 0) return AMGB_OK;
        scale_kernel<<<vec_grid(S, n), 256, 0, stream>>>(a, x, y, n);
        CK(cudaGetLastError());
        launches++;
        return AMGB_OK;
    }
    int normal_equations(Level &L, const Smoother &s);     // jacobi_ne / gauss_seidel_ne / gauss_seidel_nr
    int schwarz(Level &L, const Smoother &s);
    int block_gauss_seidel(Level &L, const Smoother &s);   // defined below (needs its kernel)
    int block_jacobi_indexed(Level &L, const Smoother &s, const int *brows, long long m);

    // one launch = the whole smoother application (resident_kernel.cuh)
    int resident_apply(Level &L, const Smoother &s)
    {
        ResidentArgs a;
        a.n = L.A.n_rows; a.log2m = s.res_log2m; a.Ap = L.A.Ap; a.Aj = L.A.Aj; a.Ax = L.A.Ax;
        a.x = L.x; a.b = L.b; a.omega = (s.sweep == AMGB_SWEEP_SYMMETRIC) ? 1.0 : s.omega;
        a.wave_ptr = s.res_wave_ptr; a.seq = s.res_seq; a.seq_len = s.res_seq_len; a.G = L.A.lanes;
        launches++;
        RET(prof_begin(7, s.res_csize, L.A.n_rows, L.A.nnz, s.res_bytes));
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)s.res_csize);
        cfg.blockDim = dim3(kResidentThreads);
        cfg.dynamicSmemBytes = sizeof(double) << s.res_log2m;
        cfg.stream = stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)s.res_csize; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        CK(cudaLaunchKernelEx(&cfg, resident_gs_kernel, a));
        return prof_end();
    }

    // decide whether a Gauss-Seidel smoother of this level can run resident, and upload its schedule
    int resident_prepare(Level &L, Smoother &s)
    {
        if (!S.use_resident || s.kind != AMGB_SM_GAUSS_SEIDEL || !s.ws.contiguous) return AMGB_OK;
        const long long nw = (long long)s.ws.ptr.size() - 1;
        if (nw < 1 || L.A.n_rows < 1) return AMGB_OK;
        // only where the dependent-wave latency, not the operator stream, is the cost: one cluster pulls
        // the operator through 16 SMs, so bigger levels stay on the full-grid wave launches
        if (L.A.n_rows > S.resident_max_rows) return AMGB_OK;
        // largest cluster the device co-schedules with the slice it then needs in shared memory
        for (int c = 16; c >= 2; c >>= 1) {
            int log2m = 5;
            while ((1LL << log2m) * c < L.A.n_rows) log2m++;
            if (log2m > kResidentMaxLog2m) break;          // even 16 CTAs x 128 KB cannot hold x
            const size_t smem = sizeof(double) << log2m;
            CK(cudaFuncSetAttribute(resident_gs_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
            CK(cudaFuncSetAttribute(resident_gs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(128 * 1024)));
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((unsigned)c); cfg.blockDim = dim3(kResidentThreads); cfg.dynamicSmemBytes = smem;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = (unsigned)c; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
            cfg.attrs = at; cfg.numAttrs = 1;
            int ncl = 0;
            if (cudaOccupancyMaxActiveClusters(&ncl, resident_gs_kernel, &cfg) != cudaSuccess || ncl < 1) {
                cudaGetLastError();
                continue;
            }
            std::vector<int> seq;
            double bytes = 0.0;
            for (int it = 0; it < s.iterations; it++) {
                if (s.sweep == AMGB_SWEEP_FORWARD || s.sweep == AMGB_SWEEP_SYMMETRIC)
                    for (long long w = 0; w < nw; w++) seq.push_back((int)w);
                if (s.sweep == AMGB_SWEEP_BACKWARD)
                    for (long long w = nw - 1; w >= 0; w--) seq.push_back((int)w);
                if (s.sweep == AMGB_SWEEP_SYMMETRIC)
                    for (long long w = nw - 2; w >= 0; w--) seq.push_back((int)w);     // idempotent middle wave skipped
            }
            for (int w : seq)
                bytes += 12.0 * s.ws.nnz[(size_t)w] + 36.0 * (double)(s.ws.ptr[(size_t)w + 1] - s.ws.ptr[(size_t)w]);
            RET(upload(&s.res_wave_ptr, s.ws.ptr.data(), (long long)s.ws.ptr.size()));
            RET(upload(&s.res_seq, seq.data(), (long long)seq.size()));
            s.res_seq_len = (int)seq.size();
            s.res_log2m = log2m;
            s.res_csize = c;
            s.res_bytes = bytes;
            return AMGB_OK;
        }
        return AMGB_OK;
    }

    int coarse_solve(Level &Lc)
    {
        if (coarse_zero) return launch_count_fill(Lc.x, Lc.A.n_rows);
        if (coarse_relax) {                                             // :773-779
            Lc.x = Lc.x_home;
            RET(launch_count_fill(Lc.x, Lc.A.n_rows));
            RET(smooth(Lc, coarse_sm));
            if (Lc.x != Lc.x_home) {                                    // odd number of Jacobi ping-pongs
                if (recording) {
                    RET(record(T_COPY, 1, 0, Lc.A.n_rows, nullptr, nullptr, Lc.x, nullptr, Lc.x_home, 0.0, 16.0 * Lc.A.n_rows));
                } else {
                    RET(copy_vec(Lc.x_home, Lc.x, Lc.A.n_rows));
                }
                std::swap(Lc.x, Lc.xalt);
            }
            return AMGB_OK;
        }
        const int n = coarse_n;
        if (recording)
            return record(T_DENSE, 32, 0, n, nullptr, nullptr, Lc.b, nullptr, Lc.x, 0.0, 8.0 * n * n + 16.0 * n,
                          coarse_pinv, n);
        const int threads = 128, rows_per_block = threads / 32;
        dense_matvec_kernel<<<(n + rows_per_block - 1) / rows_per_block, threads, 0, stream>>>(
            n, n, coarse_pinv, Lc.b, Lc.x);
        CK(cudaGetLastError());
        launches++;
        return AMGB_OK;
    }

    int launch_count_fill(double *x, long long n)
    {
        if (recording) return n > 0 ? record(T_FILL, 1, 0, (int)n, nullptr, nullptr, nullptr, nullptr, x, 0.0, 8.0 * n) : AMGB_OK;
        launches += (n > 0);
        return launch_fill(S, x, n, 0.0, stream);
    }

    int launch_fill_value(double *x, long long n, double v)
    {
        launches += (n > 0);
        return launch_fill(S, x, n, v, stream);
    }

    // MultilevelSolver.__solve (multilevel.py:584-662)
    // from_zero: the level's x was just filled with +0 (the first visit after descend's fill)
    int cycle(int lvl, int kind, int cpl, bool from_zero = false)
    {
        Level &L = levels[(size_t)lvl];
        Level &C = levels[(size_t)lvl + 1];
        cur_level = lvl;
        RET(smooth_residual(L, L.pre, nullptr, nullptr, from_zero));    // :610-612
        RET(spmv(OP_SPMV, L.R, L.r, nullptr, C.b));                     // :614
        if (lvl + 1 >= tail_level && !recording && kind != AMGB_CYCLE_AMLI) RET(run_tail(lvl, kind, cpl));
        else RET(descend(lvl, kind, cpl));
        cur_level = lvl;
        RET(spmv(OP_PADD, L.P, C.x, nullptr, L.x));                     // :660
        if (lvl == 0 && fuse_stop) RET(smooth_residual(L, L.post, partials, &stop_nparts));   // :662 + :567
        else RET(smooth(L, L.post));                                    // :662
        if (L.x != L.x_home) {   // odd number of Jacobi ping-pongs: bring the iterate home
            if (recording) {
                RET(record(T_COPY, 1, 0, L.A.n_rows, nullptr, nullptr, L.x, nullptr, L.x_home, 0.0, 16.0 * L.A.n_rows));
            } else {
                CK(cudaMemcpyAsync(L.x_home, L.x, sizeof(double) * (size_t)L.A.n_rows,
                                   cudaMemcpyDeviceToDevice, stream));
                launches++;
            }
            std::swap(L.x, L.xalt);
        }
        return AMGB_OK;
    }

    // everything between restriction and prolongation at level lvl (multilevel.py:615-656)
    int descend(int lvl, int kind, int cpl)
    {
        Level &C = levels[(size_t)lvl + 1];
        if (lvl == (int)levels.size() - 2) return coarse_solve(C);      // :617-618
        if (kind == AMGB_CYCLE_AMLI) return descend_amli(lvl, cpl);     // :631-657
        RET(launch_count_fill(C.x, C.A.n_rows));                        // :615
        if (kind == AMGB_CYCLE_V) {
            RET(cycle(lvl + 1, AMGB_CYCLE_V, 1, true));                 // :619-620
        } else if (kind == AMGB_CYCLE_W) {
            RET(cycle(lvl + 1, kind, cpl, true));                       // :621-623
            RET(cycle(lvl + 1, kind, cpl));
        } else if (kind == AMGB_CYCLE_F) {
            RET(cycle(lvl + 1, kind, cpl, true));                       // :624-627
            for (int q = 0; q < cpl; q++) RET(cycle(lvl + 1, AMGB_CYCLE_V, 1));
        } else {
            return fail(AMGB_EINVAL, "Unrecognized cycle type");        // :658 (TypeError)
        }
        return AMGB_OK;
    }

    // device dot product into a device scalar (two-stage, fixed grid: bit-reproducible)
    int dot_to(const double *x, const double *y, long long n, double *out_dev)
    {
        dot_partials_kernel<<<sumsq_blocks(S), 256, 0, stream>>>(x, y, n, sumsq_parts);
        CK(cudaGetLastError());
        reduce_partials_kernel<<<1, 1024, 0, stream>>>(sumsq_parts, sumsq_blocks(S), out_dev);
        CK(cudaGetLastError());
        launches += 2;
        return AMGB_OK;
    }
    int axpy_ratio(double *y, const double *x, const double *num, const double *den, double sign, long long n)
    {
        if (n <= 0) return AMGB_OK;
        axpy_ratio_kernel<<<vec_grid(S, n), 256, 0, stream>>>(y, x, num, den, sign, n);
        CK(cudaGetLastError());
        launches++;
        return AMGB_OK;
    }
    int copy_vec(double *dst, const double *src, long long n)
    {
        CK(cudaMemcpyAsync(dst, src, sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, stream));
        launches++;
        return AMGB_OK;
    }

    // buffers of the AMLI recursion on levels 1 .. L-2 (must exist before a graph capture starts)
    int prepare_amli()
    {
        for (size_t l = 1; l + 1 < levels.size(); l++) {
            Level &C = levels[l];
            if (C.amli_s != nullptr) continue;
            const long long n = C.A.n_rows;
            RET(dalloc(&C.amli_p[0], n + 2));
            RET(dalloc(&C.amli_p[1], n + 2));
            RET(dalloc(&C.amli_Ap, n + 2));
            RET(dalloc(&C.amli_x, n + 2));
            RET(dalloc(&C.amli_s, 8));
        }
        return AMGB_OK;
    }

    // multilevel.py:631-657.  nAMLI = 2 corrections p_k = (one AMLI cycle on level lvl+1 from the all-ones guess,
    // for the CURRENT coarse rhs), A_c-orthogonalised against the earlier one, each with the optimal step
    // alpha_k = <p_k, b_c> / <p_k, A_c p_k>; the coarse rhs is updated in between.  <p_0, A_c p_0> is needed
    // twice by the reference (step size, then the orthogonalisation coefficient): computed once here.
    int descend_amli(int lvl, int cpl)
    {
        Level &C = levels[(size_t)lvl + 1];
        const long long n = C.A.n_rows;
        if (C.amli_s == nullptr) return fail(AMGB_ESTATE, "AMLI buffers not prepared");
        double *s = C.amli_s;               // s[0] = <p0,b>, s[1] = <p0,Ap0>, s[2] = <p0,A p1'>, s[3] = <p1,b>, s[4] = <p1,Ap1>
        RET(launch_count_fill(C.amli_x, n));                            // coarse_x = 0 (:615)
        for (int k = 0; k < 2; k++) {
            double *pk = C.amli_p[k];
            RET(launch_fill_value(C.x, n, 1.0));                        // p[k, :] = 1 (:640)
            RET(cycle(lvl + 1, AMGB_CYCLE_AMLI, cpl));                  // :641-642
            cur_level = lvl + 1;
            RET(copy_vec(pk, C.x, n));
            if (k == 1) {                                               // :645-648
                RET(spmv(OP_SPMV, C.A, pk, nullptr, C.amli_Ap));
                RET(dot_to(C.amli_p[0], C.amli_Ap, n, s + 2));
                RET(axpy_ratio(pk, C.amli_p[0], s + 2, s + 1, -1.0, n));
            }
            RET(spmv(OP_SPMV, C.A, pk, nullptr, C.amli_Ap));            // :651
            RET(dot_to(pk, C.b, n, s + (k == 0 ? 0 : 3)));              // :652-653
            RET(dot_to(pk, C.amli_Ap, n, s + (k == 0 ? 1 : 4)));
            RET(axpy_ratio(C.amli_x, pk, s + (k == 0 ? 0 : 3), s + (k == 0 ? 1 : 4), 1.0, n));      // :656
            RET(axpy_ratio(C.b, C.amli_Ap, s + (k == 0 ? 0 : 3), s + (k == 0 ? 1 : 4), -1.0, n));   // :659
        }
        return copy_vec(C.x, C.amli_x, n);                              // what the prolongation reads
    }

    // the same, for levels >= tail_level: recorded once, replayed by one cluster kernel
    int ensure_tail_prog(int lvl, int kind, int cpl)
    {
        TailProg &tp = tail_prog[kind];
        if (tp.dev == nullptr || tp.cpl != cpl || tp.lvl != lvl) {
            recording = true;
            rec.clear();
            rec_bytes = 0.0;
            const int rc = descend(lvl, kind, cpl);
            recording = false;
            if (rc != AMGB_OK) return rc;
            RET(upload(&tp.dev, rec.data(), (long long)rec.size()));
            tp.n = (int)rec.size(); tp.cpl = cpl; tp.lvl = lvl; tp.bytes = rec_bytes;
            rec.clear();
        }
        return AMGB_OK;
    }

    // programs must exist before a graph capture starts (recording allocates and copies)
    int prepare_tail(int kind, int cpl)
    {
        if (tail_level >= (int)levels.size()) return AMGB_OK;
        RET(ensure_tail_prog(tail_level - 1, kind, cpl));
        if (kind == AMGB_CYCLE_F) RET(ensure_tail_prog(tail_level - 1, AMGB_CYCLE_V, 1));
        return AMGB_OK;
    }

    int run_tail(int lvl, int kind, int cpl)
    {
        TailProg &tp = tail_prog[kind];
        if (tp.dev == nullptr || tp.cpl != cpl || tp.lvl != lvl)
            return fail(AMGB_ESTATE, "coarse tail program not prepared");
        if (tp.n == 0) return AMGB_OK;
        launches++;
        cur_level = lvl + 1;
        if (S.tail_grid) {
            RET(prof_begin(10, S.grid_ctas, tp.n, 0, tp.bytes));
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((unsigned)S.grid_ctas);
            cfg.blockDim = dim3(kGridThreads);
            cfg.stream = stream;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeCooperative;
            at[0].val.cooperative = 1;
            cfg.attrs = at; cfg.numAttrs = 1;
            const TailStep *prog = tp.dev;
            int nsteps = tp.n;
            GridSync *gs = grid_sync;
            CK(cudaLaunchKernelEx(&cfg, coarse_grid_kernel, prog, nsteps, gs));
            return prof_end();
        }
        RET(prof_begin(6, tail_csize, tp.n, 0, tp.bytes));
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)tail_csize);
        cfg.blockDim = dim3(kTailThreads);
        cfg.stream = stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)tail_csize; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        const TailStep *prog = tp.dev;
        int nsteps = tp.n;
        CK(cudaLaunchKernelEx(&cfg, tail_kernel, prog, nsteps));
        return prof_end();
    }

    // ||b - A x||^2 on level 0 -> norms2[slot]   (multilevel.py:545, :567 with the norm fused)
    int residual_norm2(int slot)
    {
        Level &L = levels[0];
        cur_level = 0;
        RET(spmv(OP_RESID, L.A, L.x, L.b, L.r, 0.0, nullptr, partials));
        reduce_partials_kernel<<<1, 1024, 0, stream>>>(partials, (int)partials_used(L.A, OP_RESID), norms2 + slot);
        CK(cudaGetLastError());
        launches++;
        return AMGB_OK;
    }

    // stop = true (only when stop_fusable()): the level-0 post-smoother is followed by the stop test's residual inside
    // the cycle, its |r|^2 partials left in `partials` (stop_nparts of them)
    int one_iteration(int kind, int cpl, bool stop = false)
    {
        if (levels.size() == 1) {   // multilevel.py:559-561: x = coarse_solver(A, b)
            return coarse_solve(levels[0]);
        }
        if (kind == AMGB_CYCLE_AMLI) RET(prepare_amli());
        else RET(prepare_tail(kind, cpl));
        struct StopScope {          // fuse_stop holds while the cycle below is issued or captured
            bool &f;
            StopScope(bool &f_, bool v) : f(f_) { f = v; }
            ~StopScope() { f = false; }
        } scope(fuse_stop, stop);
        if (!S.use_graph) return cycle(0, kind, cpl);
        {   // the caller is capturing this stream into ITS OWN graph (the multi-GPU layer captures the whole distributed
            // cycle): an executable graph cannot be launched into a capturing stream -- issue the launch sequence itself
            cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
            if (cudaStreamIsCapturing(stream, &st) == cudaSuccess && st == cudaStreamCaptureStatusActive)
                return cycle(0, kind, cpl);
        }
        cudaGraphExec_t *gx = stop ? graph_stop : graph;
        int *gcpl = stop ? graph_stop_cpl : graph_cpl;
        long long *gnodes = stop ? graph_stop_nodes : graph_nodes;
        if (gx[kind] == nullptr || gcpl[kind] != cpl) {
            if (gx[kind] != nullptr) { cudaGraphExecDestroy(gx[kind]); gx[kind] = nullptr; }
            const long long before = launches;
            cudaGraph_t g = nullptr;
            CK(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
            int rc = cycle(0, kind, cpl);
            cudaError_t e = cudaStreamEndCapture(stream, &g);
            if (rc != AMGB_OK) { if (g) cudaGraphDestroy(g); return rc; }
            if (e != cudaSuccess) return fail(AMGB_ECUDA, std::string("graph capture: ") + cudaGetErrorString(e));
            gnodes[kind] = launches - before;
            launches = before;
            CK(cudaGraphInstantiate(&gx[kind], g, 0));
            cudaGraphDestroy(g);
            gcpl[kind] = cpl;
        }
        CK(cudaGraphLaunch(gx[kind], stream));
        launches += gnodes[kind];
        return AMGB_OK;
    }

    // the stop test's residual can ride on the level-0 post-smoother's last wave
    bool stop_fusable() const { return levels.size() > 1 && resid_wave(levels[0], levels[0].post, true) >= 0; }

    // one cycle, then ||b - A x||^2 on level 0 into norms2[slot] (multilevel.py:559-567)
    int iteration_norm2(int kind, int cpl, int slot)
    {
        if (!stop_fusable()) {
            RET(one_iteration(kind, cpl));
            return residual_norm2(slot);
        }
        RET(one_iteration(kind, cpl, true));
        reduce_partials_kernel<<<1, 1024, 0, stream>>>(partials, (int)stop_nparts, norms2 + slot);
        CK(cudaGetLastError());
        launches++;
        return AMGB_OK;
    }

    int ensure_norms(int need)
    {
        if (need <= norms2_cap) return AMGB_OK;
        int cap = std::max(need, 128);
        RET(dalloc(&norms2, cap));
        norms2_cap = cap;
        return AMGB_OK;
    }

    // level-0 vectors live in wave-major order: dst[i] = src[idx[i]]
    int gather(const double *src, const int *idx, double *dst, long long n)
    {
        if (n <= 0) return AMGB_OK;
        gather_kernel<<<vec_grid(S, n), 256, 0, stream>>>(src, idx, dst, n);
        CK(cudaGetLastError());
        launches++;
        return AMGB_OK;
    }

    int make_smoother(const SmootherSpec &sp, const HostCsr &Aperm, const std::vector<int> *pos,
                      const WaveSchedule *shared, Smoother &s);
    int prepare_zero_start(const HostCsr &A, const WaveSchedule &W, Level &L);
    void plan_layout(const HostLevel &H, LevelLayout &Y) const;
    int build_level(int l, const HostLevel &H, LevelLayout &Y, const LevelLayout *next);
    int finalize_levels();
};

// ------------------------------------------------------------------------------------------
// block Jacobi (relaxation.h:1021-1090) on the point-CSR expansion of a BSR operator:
// one group of G lanes per BLOCK row; for each of its bs point rows the off-block-diagonal
// products are summed (entries whose column block equals the row block are skipped, exactly
// the `if (i == j) continue` of the reference), then x_I = (1-w) x_I + w Dinv_I (b_I - rsum).
// ------------------------------------------------------------------------------------------
template <int G, int BS>
__global__ void __launch_bounds__(kCsrThreads) block_jacobi_kernel(int nb, const int *__restrict__ Ap,
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
    double rs[BS];
#pragma unroll
    for (int k = 0; k < BS; k++) {
        double sum = 0.0;
        if (active) {
            const int row = (int)I * BS + k;
            const int s = Ap[row], e = Ap[row + 1];
            for (int jj = s + lane; jj < e; jj += G) {
                const int c = ld_stream_i32(Aj + jj);
                const double v = ld_stream_f64(Ax + jj);
                if (c / BS != (int)I) sum += v * __ldg(x + c);
            }
        }
        rs[k] = group_sum<G>(sum);
    }
    if (active && lane == 0) {
        const size_t base = (size_t)I * BS;
#pragma unroll
        for (int k = 0; k < BS; k++) rs[k] = b[base + k] - rs[k];
#pragma unroll
        for (int k = 0; k < BS; k++) {
            double v = 0.0;
#pragma unroll
            for (int c = 0; c < BS; c++) v += Dinv[base * BS + (size_t)k * BS + c] * rs[c];
            y[base + k] = (1.0 - omega) * x[base + k] + omega * v;
        }
    }
}

template <int BS>
static int launch_block_jacobi(int lanes, int nb, const DevCsr &A, const double *x, const double *b,
                               const double *Dinv, double *y, double omega, cudaStream_t s)
{
    if (nb <= 0) return AMGB_OK;
    const dim3 g((unsigned)csr_grid(nb, lanes)), t(kCsrThreads);
    switch (lanes) {
    case 1: block_jacobi_kernel<1, BS><<<g, t, 0, s>>>(nb, A.Ap, A.Aj, A.Ax, x, b, Dinv, y, omega); break;
    case 2: block_jacobi_kernel<2, BS><<<g, t, 0, s>>>(nb, A.Ap, A.Aj, A.Ax, x, b, Dinv, y, omega); break;
    case 4: block_jacobi_kernel<4, BS><<<g, t, 0, s>>>(nb, A.Ap, A.Aj, A.Ax, x, b, Dinv, y, omega); break;
    case 8: block_jacobi_kernel<8, BS><<<g, t, 0, s>>>(nb, A.Ap, A.Aj, A.Ax, x, b, Dinv, y, omega); break;
    case 16: block_jacobi_kernel<16, BS><<<g, t, 0, s>>>(nb, A.Ap, A.Aj, A.Ax, x, b, Dinv, y, omega); break;
    default: block_jacobi_kernel<32, BS><<<g, t, 0, s>>>(nb, A.Ap, A.Aj, A.Ax, x, b, Dinv, y, omega); break;
    }
    CK(cudaGetLastError());
    return AMGB_OK;
}

static int dispatch_block_jacobi(int bs, int lanes, int nb, const DevCsr &A, const double *x,
                                 const double *b, const double *Dinv, double *y, double omega,
                                 cudaStream_t s)
{
    switch (bs) {
    case 1: return launch_block_jacobi<1>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 2: return launch_block_jacobi<2>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 3: return launch_block_jacobi<3>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 4: return launch_block_jacobi<4>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 5: return launch_block_jacobi<5>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 6: return launch_block_jacobi<6>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 7: return launch_block_jacobi<7>(lanes, nb, A, x, b, Dinv, y, omega, s);
    case 8: return launch_block_jacobi<8>(lanes, nb, A, x, b, Dinv, y, omega, s);
    }
    return fail(AMGB_ENOTIMPL, "block_jacobi: blocksize must be 1..8");
}

int amgb_hierarchy::block_jacobi(Level &L, const Smoother &s)
{
    const int nb = L.A.n_rows / s.bs;
    for (int it = 0; it < s.iterations; it++) {
        if (recording) return fail(AMGB_ESTATE, "block Jacobi inside the cluster tail");
        RET(prof_begin(5, L.A.lanes, L.A.n_rows, L.A.nnz,
                       12.0 * L.A.nnz + 4.0 * (L.A.n_rows + 1) + (24.0 + 8.0 * s.bs) * L.A.n_rows));
        RET(dispatch_block_jacobi(s.bs, L.A.lanes, nb, L.A, L.x, L.b, s.Dinv, L.xalt, s.omega, stream));
        RET(prof_end());
        launches++;
        std::swap(L.x, L.xalt);
    }
    return AMGB_OK;
}

// ------------------------------------------------------------------------------------------
// block Gauss-Seidel (relaxation.h:1242-1298) on the point-CSR expansion: the sequential sweep over block
// rows is executed in dependency waves of the BLOCK graph (build_waves on the block pattern); inside a wave
// one group of G lanes per block row sums the off-diagonal-block products with the CURRENT iterate and
// writes x_I = Dinv_I (b_I - rsum) in place (no block of the wave reads another block of the same wave).
// ------------------------------------------------------------------------------------------
template <int G, int BS>
__global__ void __launch_bounds__(kCsrThreads) block_gs_kernel(int nrows, const int *__restrict__ brows,
                                                               const int *__restrict__ Ap, const int *__restrict__ Aj,
                                                               const double *__restrict__ Ax, double *x,
                                                               const double *__restrict__ b,
                                                               const double *__restrict__ Dinv)
{
    const int lane = threadIdx.x & (G - 1);
    const long long k = ((long long)blockIdx.x * kCsrThreads + threadIdx.x) / G;
    const bool active = k < nrows;
    const int I = active ? brows[k] : 0;
    double rs[BS];
#pragma unroll
    for (int q = 0; q < BS; q++) {
        double sum = 0.0;
        if (active) {
            const int row = I * BS + q;
            const int s = Ap[row], e = Ap[row + 1];
            for (int jj = s + lane; jj < e; jj += G) {
                const int c = ld_stream_i32(Aj + jj);
                const double v = ld_stream_f64(Ax + jj);
                if (c / BS != I) sum += v * x[c];           // plain load: x is written by this launch
            }
        }
        rs[q] = group_sum<G>(sum);
    }
    if (active && lane == 0) {
        const size_t base = (size_t)I * BS;
#pragma unroll
        for (int q = 0; q < BS; q++) rs[q] = b[base + q] - rs[q];
#pragma unroll
        for (int q = 0; q < BS; q++) {
            double v = 0.0;
#pragma unroll
            for (int c = 0; c < BS; c++) v += Dinv[base * BS + (size_t)q * BS + c] * rs[c];
            x[base + q] = v;
        }
    }
}

template <int BS>
static int launch_block_gs(int lanes, int nrows, const int *brows, const DevCsr &A, double *x, const double *b,
                           const double *Dinv, cudaStream_t s)
{
    if (nrows <= 0) return AMGB_OK;
    const dim3 g((unsigned)csr_grid(nrows, lanes)), t(kCsrThreads);
    switch (lanes) {
    case 1: block_gs_kernel<1, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, x, b, Dinv); break;
    case 2: block_gs_kernel<2, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, x, b, Dinv); break;
    case 4: block_gs_kernel<4, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, x, b, Dinv); break;
    case 8: block_gs_kernel<8, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, x, b, Dinv); break;
    case 16: block_gs_kernel<16, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, x, b, Dinv); break;
    default: block_gs_kernel<32, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, x, b, Dinv); break;
    }
    CK(cudaGetLastError());
    return AMGB_OK;
}

static int dispatch_block_gs(int bs, int lanes, int nrows, const int *brows, const DevCsr &A, double *x,
                             const double *b, const double *Dinv, cudaStream_t s)
{
    switch (bs) {
    case 1: return launch_block_gs<1>(lanes, nrows, brows, A, x, b, Dinv, s);
    case 2: return launch_block_gs<2>(lanes, nrows, brows, A, x, b, Dinv, s);
    case 3: return launch_block_gs<3>(lanes, nrows, brows, A, x, b, Dinv, s);
    case 4: return launch_block_gs<4>(lanes, nrows, brows, A, x, b, Dinv, s);
    case 5: return launch_block_gs<5>(lanes, nrows, brows, A, x, b, Dinv, s);
    case 6: return launch_block_gs<6>(lanes, nrows, brows, A, x, b, Dinv, s);
    case 7: return launch_block_gs<7>(lanes, nrows, brows, A, x, b, Dinv, s);
    case 8: return launch_block_gs<8>(lanes, nrows, brows, A, x, b, Dinv, s);
    }
    return fail(AMGB_ENOTIMPL, "block_gauss_seidel: blocksize must be 1..8");
}

// indexed block Jacobi (relaxation.h:1113-1172): the listed block rows are relaxed from the snapshot `xold`
template <int G, int BS>
__global__ void __launch_bounds__(kCsrThreads) block_jacobi_indexed_kernel(int nrows, const int *__restrict__ brows,
                                                                           const int *__restrict__ Ap, const int *__restrict__ Aj,
                                                                           const double *__restrict__ Ax,
                                                                           const double *__restrict__ xold,
                                                                           const double *__restrict__ b,
                                                                           const double *__restrict__ Dinv,
                                                                           double *__restrict__ x, double omega)
{
    const int lane = threadIdx.x & (G - 1);
    const long long k = ((long long)blockIdx.x * kCsrThreads + threadIdx.x) / G;
    const bool active = k < nrows;
    const int I = active ? brows[k] : 0;
    double rs[BS];
#pragma unroll
    for (int q = 0; q < BS; q++) {
        double sum = 0.0;
        if (active) {
            const int row = I * BS + q;
            const int s = Ap[row], e = Ap[row + 1];
            for (int jj = s + lane; jj < e; jj += G) {
                const int c = ld_stream_i32(Aj + jj);
                const double v = ld_stream_f64(Ax + jj);
                if (c / BS != I) sum += v * __ldg(xold + c);
            }
        }
        rs[q] = group_sum<G>(sum);
    }
    if (active && lane == 0) {
        const size_t base = (size_t)I * BS;
#pragma unroll
        for (int q = 0; q < BS; q++) rs[q] = b[base + q] - rs[q];
#pragma unroll
        for (int q = 0; q < BS; q++) {
            double v = 0.0;
#pragma unroll
            for (int c = 0; c < BS; c++) v += Dinv[base * BS + (size_t)q * BS + c] * rs[c];
            x[base + q] = (1.0 - omega) * xold[base + q] + omega * v;
        }
    }
}

template <int BS>
static int launch_block_jacobi_indexed(int lanes, int nrows, const int *brows, const DevCsr &A, const double *xold,
                                       const double *b, const double *Dinv, double *x, double omega, cudaStream_t s)
{
    if (nrows <= 0) return AMGB_OK;
    const dim3 g((unsigned)csr_grid(nrows, lanes)), t(kCsrThreads);
    switch (lanes) {
    case 1: block_jacobi_indexed_kernel<1, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, xold, b, Dinv, x, omega); break;
    case 2: block_jacobi_indexed_kernel<2, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, xold, b, Dinv, x, omega); break;
    case 4: block_jacobi_indexed_kernel<4, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, xold, b, Dinv, x, omega); break;
    case 8: block_jacobi_indexed_kernel<8, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, xold, b, Dinv, x, omega); break;
    case 16: block_jacobi_indexed_kernel<16, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, xold, b, Dinv, x, omega); break;
    default: block_jacobi_indexed_kernel<32, BS><<<g, t, 0, s>>>(nrows, brows, A.Ap, A.Aj, A.Ax, xold, b, Dinv, x, omega); break;
    }
    CK(cudaGetLastError());
    return AMGB_OK;
}

int amgb_hierarchy::block_jacobi_indexed(Level &L, const Smoother &s, const int *brows, long long m)
{
    if (recording) return fail(AMGB_ESTATE, "indexed block Jacobi inside the cluster tail");
    if (m <= 0) return AMGB_OK;
    double *temp = (L.x == L.x_home) ? L.xalt : L.x_home;
    RET(copy_vec(temp, L.x, L.A.n_rows));
    launches++;
    RET(prof_begin(8, L.A.lanes, m * s.bs, 0, 16.0 * L.A.n_rows + (4.0 + (24.0 + 8.0 * s.bs) * s.bs) * (double)m));
    switch (s.bs) {
    case 2: RET(launch_block_jacobi_indexed<2>(L.A.lanes, (int)m, brows, L.A, temp, L.b, s.Dinv, L.x, s.omega, stream)); break;
    case 3: RET(launch_block_jacobi_indexed<3>(L.A.lanes, (int)m, brows, L.A, temp, L.b, s.Dinv, L.x, s.omega, stream)); break;
    case 4: RET(launch_block_jacobi_indexed<4>(L.A.lanes, (int)m, brows, L.A, temp, L.b, s.Dinv, L.x, s.omega, stream)); break;
    case 5: RET(launch_block_jacobi_indexed<5>(L.A.lanes, (int)m, brows, L.A, temp, L.b, s.Dinv, L.x, s.omega, stream)); break;
    case 6: RET(launch_block_jacobi_indexed<6>(L.A.lanes, (int)m, brows, L.A, temp, L.b, s.Dinv, L.x, s.omega, stream)); break;
    case 7: RET(launch_block_jacobi_indexed<7>(L.A.lanes, (int)m, brows, L.A, temp, L.b, s.Dinv, L.x, s.omega, stream)); break;
    case 8: RET(launch_block_jacobi_indexed<8>(L.A.lanes, (int)m, brows, L.A, temp, L.b, s.Dinv, L.x, s.omega, stream)); break;
    default: RET(launch_block_jacobi_indexed<1>(L.A.lanes, (int)m, brows, L.A, temp, L.b, s.Dinv, L.x, s.omega, stream)); break;
    }
    return prof_end();
}

// ------------------------------------------------------------------------------------------
// normal-equation smoothers
// ------------------------------------------------------------------------------------------
static void sort_rows_by_column(HostCsr &A)       // what scipy's sort_indices does (util.get_diagonal sorts in place)
{
    std::vector<std::pair<int, double>> row;
    for (int i = 0; i < A.n_rows; i++) {
        const int s = A.Ap[(size_t)i], e = A.Ap[(size_t)i + 1];
        row.resize((size_t)(e - s));
        for (int jj = s; jj < e; jj++) row[(size_t)(jj - s)] = {A.Aj[(size_t)jj], A.Ax[(size_t)jj]};
        std::stable_sort(row.begin(), row.end(), [](const std::pair<int, double> &a, const std::pair<int, double> &b) { return a.first < b.first; });
        for (int jj = s; jj < e; jj++) { A.Aj[(size_t)jj] = row[(size_t)(jj - s)].first; A.Ax[(size_t)jj] = row[(size_t)(jj - s)].second; }
    }
}

static void transpose_csr(const HostCsr &A, HostCsr &T)     // rows of T = columns of A, entries by ascending row of A
{
    T.n_rows = A.n_cols; T.n_cols = A.n_rows;
    T.Ap.assign((size_t)A.n_cols + 1, 0);
    T.Aj.resize(A.Aj.size());
    T.Ax.resize(A.Ax.size());
    for (int c : A.Aj) T.Ap[(size_t)c + 1]++;
    for (int c = 0; c < A.n_cols; c++) T.Ap[(size_t)c + 1] += T.Ap[(size_t)c];
    std::vector<int> cur(T.Ap.begin(), T.Ap.end() - 1);
    for (int i = 0; i < A.n_rows; i++)
        for (int jj = A.Ap[(size_t)i]; jj < A.Ap[(size_t)i + 1]; jj++) {
            const int p = cur[(size_t)A.Aj[(size_t)jj]]++;
            T.Aj[(size_t)p] = i;
            T.Ax[(size_t)p] = A.Ax[(size_t)jj];
        }
}

// sequential sweep over the rows 0..n-1 of M, each reading AND writing the vector entries of its columns: row i goes
// to wave 1 + (latest wave that touched any of its columns); waves in order == the sequential sweep, in reverse
// order == the backward sweep
static bool build_conflict_waves(const HostCsr &M, std::vector<int> &rows_sorted, std::vector<long long> &ptr)
{
    std::vector<int> last((size_t)M.n_cols, 0), w((size_t)M.n_rows);
    std::vector<int> seen((size_t)M.n_cols, -1);
    int maxw = 0;
    for (int i = 0; i < M.n_rows; i++) {
        int wv = 0;
        for (int jj = M.Ap[(size_t)i]; jj < M.Ap[(size_t)i + 1]; jj++) {
            const int c = M.Aj[(size_t)jj];
            if (seen[(size_t)c] == i) return false;            // duplicate column in a row: lanes would collide
            seen[(size_t)c] = i;
            wv = std::max(wv, last[(size_t)c]);
        }
        wv += 1;
        w[(size_t)i] = wv;
        for (int jj = M.Ap[(size_t)i]; jj < M.Ap[(size_t)i + 1]; jj++) last[(size_t)M.Aj[(size_t)jj]] = wv;
        maxw = std::max(maxw, wv);
    }
    ptr.assign((size_t)maxw + 1, 0);
    for (int i = 0; i < M.n_rows; i++) ptr[(size_t)w[(size_t)i]]++;
    for (int q = 0; q < maxw; q++) ptr[(size_t)q + 1] += ptr[(size_t)q];
    rows_sorted.resize((size_t)M.n_rows);
    std::vector<long long> cur(ptr.begin(), ptr.end() - 1);
    for (int i = 0; i < M.n_rows; i++) rows_sorted[(size_t)cur[(size_t)w[(size_t)i] - 1]++] = i;
    return true;
}

template <bool NR>
static int launch_kaczmarz(int lanes, int nrows, const int *rows, const DevCsr &M, double *v, const double *b,
                           const double *Dinv, double omega, double *xout, cudaStream_t s)
{
    if (nrows <= 0) return AMGB_OK;
    const dim3 g((unsigned)csr_grid(nrows, lanes)), t(kCsrThreads);
    switch (lanes) {
    case 1: kaczmarz_kernel<1, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    case 2: kaczmarz_kernel<2, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    case 4: kaczmarz_kernel<4, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    case 8: kaczmarz_kernel<8, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    case 16: kaczmarz_kernel<16, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    default: kaczmarz_kernel<32, NR><<<g, t, 0, s>>>(nrows, rows, M.Ap, M.Aj, M.Ax, v, b, Dinv, omega, xout); break;
    }
    CK(cudaGetLastError());
    return AMGB_OK;
}

int amgb_hierarchy::normal_equations(Level &L, const Smoother &s)
{
    if (recording) return fail(AMGB_ESTATE, "normal-equation smoother inside the cluster tail");
    const long long n = L.A.n_rows;
    if (s.kind == AMGB_SM_JACOBI_NE) {                                   // relaxation.py:806-812
        double *temp = (L.x == L.x_home) ? L.xalt : L.x_home;
        const unsigned grid = vec_grid(S, n);
        for (int it = 0; it < s.iterations; it++) {
            RET(spmv(OP_RESID, s.ne_A, L.x, L.b, L.r));                  // b - A x
            mul_kernel<<<grid, 256, 0, stream>>>(L.r, s.Dinv, n);                // delta = (b - A x) * Dinv
            CK(cudaGetLastError());
            launches++;
            RET(spmv(OP_SPMV, s.ne_At, L.r, nullptr, temp));             // temp = (omega A^H) delta   (relaxation.h:592-600)
            RET(axpby(1.0, temp, 1.0, L.x, n));                          // x += temp                  (:602-603)
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
            launches++;
            if (nr) RET(launch_kaczmarz<true>(M.lanes, nrow, s.ws.rows + s.ws.ptr[(size_t)w], M, L.r, nullptr, s.Dinv, s.omega, L.x, stream));
            else RET(launch_kaczmarz<false>(M.lanes, nrow, s.ws.rows + s.ws.ptr[(size_t)w], M, L.x, L.b, s.Dinv, s.omega, nullptr, stream));
        }
        return AMGB_OK;
    };
    auto residual = [&]() -> int { return nr ? spmv(OP_RESID, s.ne_A, L.x, L.b, L.r) : AMGB_OK; };   // relaxation.py:992
    if (s.sweep == AMGB_SWEEP_SYMMETRIC) {                               // :883-889 / :971-977: fwd call, then bwd call
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

// multiplicative Schwarz: subdomain k reads x on the columns of its rows and writes x on its rows; it goes to wave
// 1 + (latest wave that wrote anything it reads, or read / wrote anything it writes)
static void build_schwarz_waves(const HostCsr &A, const std::vector<int> &Sj, const std::vector<int> &Sp,
                                std::vector<int> &doms_sorted, std::vector<long long> &ptr)
{
    const int nd = (int)Sp.size() - 1;
    std::vector<int> wwave((size_t)A.n_rows, 0), rwave((size_t)A.n_rows, 0), w((size_t)std::max(nd, 1));
    int maxw = 0;
    for (int k = 0; k < nd; k++) {
        int wv = 0;
        for (int q = Sp[(size_t)k]; q < Sp[(size_t)k + 1]; q++) {
            const int row = Sj[(size_t)q];
            wv = std::max(wv, std::max(rwave[(size_t)row], wwave[(size_t)row]));
            for (int jj = A.Ap[(size_t)row]; jj < A.Ap[(size_t)row + 1]; jj++) wv = std::max(wv, wwave[(size_t)A.Aj[(size_t)jj]]);
        }
        wv += 1;
        w[(size_t)k] = wv;
        for (int q = Sp[(size_t)k]; q < Sp[(size_t)k + 1]; q++) {
            const int row = Sj[(size_t)q];
            wwave[(size_t)row] = wv;
            for (int jj = A.Ap[(size_t)row]; jj < A.Ap[(size_t)row + 1]; jj++) {
                int &rw = rwave[(size_t)A.Aj[(size_t)jj]];
                rw = std::max(rw, wv);
            }
        }
        maxw = std::max(maxw, wv);
    }
    ptr.assign((size_t)maxw + 1, 0);
    for (int k = 0; k < nd; k++) ptr[(size_t)w[(size_t)k]]++;
    for (int q = 0; q < maxw; q++) ptr[(size_t)q + 1] += ptr[(size_t)q];
    doms_sorted.resize((size_t)nd);
    std::vector<long long> cur(ptr.begin(), ptr.end() - 1);
    for (int k = 0; k < nd; k++) doms_sorted[(size_t)cur[(size_t)w[(size_t)k] - 1]++] = k;
}

int amgb_hierarchy::schwarz(Level &L, const Smoother &s)
{
    if (recording) return fail(AMGB_ESTATE, "Schwarz smoother inside the cluster tail");
    const long long nw = (long long)s.ws.ptr.size() - 1;
    const size_t smem = (size_t)kSchwarzWarps * 2 * (size_t)std::max(s.sz_max_m, 1) * sizeof(double);
    auto sweep = [&](bool forward) -> int {
        for (long long q = 0; q < nw; q++) {
            const long long w = forward ? q : nw - 1 - q;
            const int nd = (int)(s.ws.ptr[(size_t)w + 1] - s.ws.ptr[(size_t)w]);
            if (nd <= 0) continue;
            schwarz_kernel<<<(unsigned)((nd + kSchwarzWarps - 1) / kSchwarzWarps), kSchwarzWarps * 32, smem, stream>>>(
                nd, s.ws.rows + s.ws.ptr[(size_t)w], s.sz_Sp, s.sz_Sj, s.sz_Tp, s.Dinv, s.ne_A.Ap, s.ne_A.Aj, s.ne_A.Ax, L.x, L.b,
                std::max(s.sz_max_m, 1));
            CK(cudaGetLastError());
            launches++;
        }
        return AMGB_OK;
    };
    for (int it = 0; it < s.iterations; it++) {                            // relaxation.py:241-262
        if (s.sweep == AMGB_SWEEP_FORWARD || s.sweep == AMGB_SWEEP_SYMMETRIC) RET(sweep(true));
        if (s.sweep == AMGB_SWEEP_BACKWARD || s.sweep == AMGB_SWEEP_SYMMETRIC) RET(sweep(false));
    }
    return AMGB_OK;
}

int amgb_hierarchy::block_gauss_seidel(Level &L, const Smoother &s)
{
    if (recording) return fail(AMGB_ESTATE, "block Gauss-Seidel inside the cluster tail");
    const long long nw = (long long)s.ws.ptr.size() - 1;
    auto wave = [&](long long w) -> int {
        const int nr = (int)(s.ws.ptr[(size_t)w + 1] - s.ws.ptr[(size_t)w]);
        if (nr <= 0) return AMGB_OK;
        launches++;
        RET(prof_begin(9, L.A.lanes, (long long)nr * s.bs, s.ws.nnz[(size_t)w],
                       12.0 * s.ws.nnz[(size_t)w] + (4.0 + (28.0 + 8.0 * s.bs) * s.bs) * nr));
        RET(dispatch_block_gs(s.bs, L.A.lanes, nr, s.ws.rows + s.ws.ptr[(size_t)w], L.A, L.x, L.b, s.Dinv, stream));
        return prof_end();
    };
    for (int it = 0; it < s.iterations; it++) {                          // relaxation.py:561-582
        if (s.sweep == AMGB_SWEEP_FORWARD || s.sweep == AMGB_SWEEP_SYMMETRIC)
            for (long long w = 0; w < nw; w++) RET(wave(w));
        if (s.sweep == AMGB_SWEEP_BACKWARD)
            for (long long w = nw - 1; w >= 0; w--) RET(wave(w));
        if (s.sweep == AMGB_SWEEP_SYMMETRIC)       // the middle wave relaxed twice in a row is idempotent: skipped
            for (long long w = nw - 2; w >= 0; w--) RET(wave(w));
    }
    return AMGB_OK;
}

// smoother on the (possibly permuted) level operator.  `pos` maps original row ids to the level's
// numbering (null = identity).  If `shared` is given the schedule is the level's own wave-major
// layout (contiguous waves); otherwise waves are derived here and executed through a row list.
int amgb_hierarchy::make_smoother(const SmootherSpec &sp, const HostCsr &Aperm, const std::vector<int> *pos,
                                  const WaveSchedule *shared, Smoother &s)
{
    s = Smoother();
    s.kind = sp.kind;
    s.iterations = sp.iterations;
    s.sweep = sp.sweep;
    s.omega = sp.omega;
    s.bs = sp.bs;
    if (sp.kind == AMGB_SM_GAUSS_SEIDEL) {
        if (shared != nullptr) {
            s.ws = *shared;
            return AMGB_OK;
        }
        std::vector<int> list;
        const int *lp = nullptr;
        long long m = Aperm.n_rows;
        if (sp.has_list) {
            list = sp.list;
            if (pos) for (int &v : list) v = (*pos)[(size_t)v];
            lp = list.data();
            m = (long long)list.size();
        } else if (pos) {            // natural order of the ORIGINAL numbering
            list.resize((size_t)Aperm.n_rows);
            for (int i = 0; i < Aperm.n_rows; i++) list[(size_t)i] = (*pos)[(size_t)i];
            lp = list.data();
        }
        std::vector<int> rows;
        build_waves(Aperm, lp, m, rows, s.ws.ptr);
        RET(upload(&s.ws.rows, rows.data(), m));
        s.ws.nnz.assign(s.ws.ptr.size() - 1, 0);
        for (size_t w = 0; w + 1 < s.ws.ptr.size(); w++)
            for (long long k = s.ws.ptr[w]; k < s.ws.ptr[w + 1]; k++)
                s.ws.nnz[w] += Aperm.Ap[(size_t)rows[(size_t)k] + 1] - Aperm.Ap[(size_t)rows[(size_t)k]];
    } else if (sp.kind == AMGB_SM_BLOCK_JACOBI) {
        RET(upload(&s.Dinv, sp.Dinv.data(), (long long)sp.Dinv.size()));
    } else if (sp.kind == AMGB_SM_POLYNOMIAL) {
        s.coef = sp.coef;
    } else if (sp.kind == AMGB_SM_JACOBI_INDEXED || sp.kind == AMGB_SM_CF_JACOBI || sp.kind == AMGB_SM_FC_JACOBI) {
        s.f_iterations = sp.f_iterations;
        s.c_iterations = sp.c_iterations;
        if (shared != nullptr) {                    // the level is stored C-points first, F-points behind them
            s.ws = *shared;
            s.cf_contig = true;
        }
        std::vector<int> l1 = sp.list, l2 = sp.list2;
        if (pos) {                                  // the level was put in wave-major order by its other smoother
            for (int &v : l1) v = (*pos)[(size_t)v];
            for (int &v : l2) v = (*pos)[(size_t)v];
        }
        RET(upload(&s.rows1, l1.data(), (long long)l1.size()));
        RET(upload(&s.rows2, l2.data(), (long long)l2.size()));
        s.n_rows1 = (long long)l1.size();
        s.n_rows2 = (long long)l2.size();
    } else if (sp.kind == AMGB_SM_JACOBI_NE || sp.kind == AMGB_SM_GAUSS_SEIDEL_NE || sp.kind == AMGB_SM_GAUSS_SEIDEL_NR) {
        if (pos) return fail(AMGB_ESTATE, "normal-equation smoother on a permuted level");
        RET(upload(&s.Dinv, sp.Dinv.data(), (long long)sp.Dinv.size(), 2));
        HostCsr As = Aperm, At;
        sort_rows_by_column(As);
        transpose_csr(As, At);
        if (sp.kind == AMGB_SM_JACOBI_NE)
            for (double &v : At.Ax) v = sp.omega * v;                    // omega2 * conjugate(Ax[j])   (relaxation.h:598)
        if (sp.kind != AMGB_SM_GAUSS_SEIDEL_NE || true) RET(upload_csr(As, s.ne_A));
        if (sp.kind != AMGB_SM_GAUSS_SEIDEL_NE) RET(upload_csr(At, s.ne_At));
        if (sp.kind != AMGB_SM_JACOBI_NE) {
            std::vector<int> rows;
            if (!build_conflict_waves(sp.kind == AMGB_SM_GAUSS_SEIDEL_NR ? At : As, rows, s.ws.ptr))
                return fail(AMGB_ENOTIMPL, "gauss_seidel_ne / _nr: duplicate column entries inside a row");
            RET(upload(&s.ws.rows, rows.data(), (long long)rows.size()));
        }
    } else if (sp.kind == AMGB_SM_SCHWARZ) {
        if (pos) return fail(AMGB_ESTATE, "Schwarz smoother on a permuted level");
        HostCsr As = Aperm;
        sort_rows_by_column(As);                                  // relaxation.py:228 (A.sort_indices())
        RET(upload_csr(As, s.ne_A));
        const std::vector<int> &Sj = sp.list, &Sp = sp.list2;
        const int nd = (int)Sp.size() - 1;
        std::vector<long long> Tp((size_t)nd + 1, 0);
        int max_m = 0;
        for (int k = 0; k < nd; k++) {
            const long long m = Sp[(size_t)k + 1] - Sp[(size_t)k];
            Tp[(size_t)k + 1] = Tp[(size_t)k] + m * m;
            max_m = std::max<int>(max_m, (int)m);
        }
        if ((long long)sp.Dinv.size() != Tp[(size_t)nd]) return fail(AMGB_EINVAL, "schwarz: inv_subblock size != sum of subdomain sizes squared");
        if ((size_t)kSchwarzWarps * 2 * (size_t)max_m * sizeof(double) > 200 * 1024) return fail(AMGB_ENOTIMPL, "schwarz: subdomain too large");
        s.sz_max_m = max_m;
        RET(upload(&s.sz_Sj, Sj.data(), (long long)Sj.size()));
        RET(upload(&s.sz_Sp, Sp.data(), (long long)Sp.size()));
        RET(upload(&s.sz_Tp, Tp.data(), (long long)Tp.size()));
        RET(upload(&s.Dinv, sp.Dinv.data(), (long long)sp.Dinv.size()));
        std::vector<int> doms;
        build_schwarz_waves(As, Sj, Sp, doms, s.ws.ptr);
        RET(upload(&s.ws.rows, doms.data(), (long long)doms.size()));
        const size_t smem = (size_t)kSchwarzWarps * 2 * (size_t)std::max(max_m, 1) * sizeof(double);
        if (smem > 48 * 1024) CK(cudaFuncSetAttribute(schwarz_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    } else if (sp.kind == AMGB_SM_CF_BLOCK_JACOBI || sp.kind == AMGB_SM_FC_BLOCK_JACOBI) {
        if (pos) return fail(AMGB_ESTATE, "block CF Jacobi on a permuted level");
        s.f_iterations = sp.f_iterations;
        s.c_iterations = sp.c_iterations;
        RET(upload(&s.Dinv, sp.Dinv.data(), (long long)sp.Dinv.size()));
        RET(upload(&s.rows1, sp.list.data(), (long long)sp.list.size()));
        RET(upload(&s.rows2, sp.list2.data(), (long long)sp.list2.size()));
        s.n_rows1 = (long long)sp.list.size();
        s.n_rows2 = (long long)sp.list2.size();
    } else if (sp.kind == AMGB_SM_BLOCK_GAUSS_SEIDEL) {
        if (pos) return fail(AMGB_ESTATE, "block Gauss-Seidel on a permuted level");
        RET(upload(&s.Dinv, sp.Dinv.data(), (long long)sp.Dinv.size()));
        // block pattern of the point expansion: block row I references block column c / bs of every entry of its
        // bs point rows (the rows of a BSR block row share one pattern; a CSR operator viewed block-wise may not)
        const int bs = sp.bs, nb = Aperm.n_rows / bs;
        HostCsr Bg;
        Bg.n_rows = Bg.n_cols = nb;
        Bg.Ap.assign((size_t)nb + 1, 0);
        std::vector<int> mark((size_t)nb, -1);
        for (int I = 0; I < nb; I++) {
            for (int jj = Aperm.Ap[(size_t)I * bs]; jj < Aperm.Ap[(size_t)(I + 1) * bs]; jj++) {
                const int J = Aperm.Aj[(size_t)jj] / bs;
                if (J < nb && mark[(size_t)J] != I) { mark[(size_t)J] = I; Bg.Aj.push_back(J); }
            }
            Bg.Ap[(size_t)I + 1] = (int)Bg.Aj.size();
        }
        std::vector<int> rows;
        build_waves(Bg, nullptr, nb, rows, s.ws.ptr);
        RET(upload(&s.ws.rows, rows.data(), (long long)rows.size()));
        s.ws.nnz.assign(s.ws.ptr.size() - 1, 0);
        for (size_t w = 0; w + 1 < s.ws.ptr.size(); w++)
            for (long long k = s.ws.ptr[w]; k < s.ws.ptr[w + 1]; k++) {
                const size_t I = (size_t)rows[(size_t)k];
                s.ws.nnz[w] += Aperm.Ap[(I + 1) * bs] - Aperm.Ap[I * bs];
            }
    }
    return AMGB_OK;
}

static bool is_permutation(const std::vector<int> &list, int n)
{
    if ((int)list.size() != n) return false;
    std::vector<char> seen((size_t)n, 0);
    for (int v : list) {
        if (v < 0 || v >= n || seen[(size_t)v]) return false;
        seen[(size_t)v] = 1;
    }
    return true;
}

// Build and upload the zero-start copy of a wave-major level operator A (already uploaded as L.A with layout W).
// Each wave is laid out for the kernel its full launch uses (gs_wave).
int amgb_hierarchy::prepare_zero_start(const HostCsr &A, const WaveSchedule &W, Level &L)
{
    const DevCsr &F = L.A;
    const size_t nw = W.ptr.size() - 1;
    if (nw < 1 || W.ptr[0] != 0 || W.ptr[nw] != A.n_rows) return AMGB_OK;
    if (F.tiles != nullptr && F.tile_G == 0) return AMGB_OK;          // flat-gather layout: full operator only
    if (!zero_start_eligible(A)) return AMGB_OK;
    ZeroStart &z = L.zs;
    z.tile.assign(nw, 0);
    for (size_t w = 0; w < nw; w++) z.tile[w] = F.tiles != nullptr && !W.tile_ptr.empty() && W.nnz[w] >= S.tile_min_nnz;
    HostCsr Z;
    build_zero_start(A, W.ptr, z.tile, F.tile_G, F.lanes, F.tile_cfg == 7 ? S.dense_T : S.tile_T, Z, z.nnz);
    return upload_csr(Z, z.A, &W.ptr, &z.tile_ptr, 0, 0, &F, S.use_value_codes);
}

// The wave-major (or C|F) row permutation of a Gauss-Seidel (or CF / FC Jacobi) level, from its pattern and smoothers
void amgb_hierarchy::plan_layout(const HostLevel &H, LevelLayout &Y) const
{
    Y = LevelLayout();
    if (!H.has_pr || !S.use_permute) return;
    // block smoothers address x in natural block numbering: such levels are never permuted
    if (H.pre.kind == AMGB_SM_BLOCK_JACOBI || H.post.kind == AMGB_SM_BLOCK_JACOBI) return;
    if (H.pre.kind == AMGB_SM_BLOCK_GAUSS_SEIDEL || H.post.kind == AMGB_SM_BLOCK_GAUSS_SEIDEL) return;
    if (H.pre.kind >= AMGB_SM_CF_BLOCK_JACOBI || H.post.kind >= AMGB_SM_CF_BLOCK_JACOBI) return;
    const SmootherSpec *src = nullptr;
    if (H.pre.kind == AMGB_SM_GAUSS_SEIDEL) { src = &H.pre; Y.src = 0; }
    else if (H.post.kind == AMGB_SM_GAUSS_SEIDEL) { src = &H.post; Y.src = 1; }
    WaveSchedule &W = Y.W;
    if (src == nullptr) {
        // CF / FC Jacobi (AIR's smoother): put the C-points first and the F-points behind them, so that a sweep
        // over either set is a contiguous row range streamed by the tile kernel instead of a row-list gather
        auto is_cf = [](int k) { return k == AMGB_SM_CF_JACOBI || k == AMGB_SM_FC_JACOBI; };
        const SmootherSpec *cf = is_cf(H.pre.kind) ? &H.pre : (is_cf(H.post.kind) ? &H.post : nullptr);
        if (cf == nullptr || !S.use_cf_layout || cf->list.empty() || cf->list2.empty()) return;
        std::vector<int> both(cf->list);
        both.insert(both.end(), cf->list2.begin(), cf->list2.end());
        if (!is_permutation(both, H.A.n_rows)) return;
        W.ptr = {0, (long long)cf->list.size(), (long long)H.A.n_rows};
        W.contiguous = true;
        W.nnz.assign(2, 0);
        for (size_t k = 0; k < both.size(); k++)
            W.nnz[k < cf->list.size() ? 0 : 1] += H.A.Ap[(size_t)both[k] + 1] - H.A.Ap[(size_t)both[k]];
        Y.order = both;
        Y.pos.resize(both.size());
        for (size_t i = 0; i < both.size(); i++) Y.pos[(size_t)both[i]] = (int)i;
        Y.src = is_cf(H.pre.kind) ? 2 : 3;                 // 2 / 3 = C|F layout taken from pre / post
        return;
    }
    if (src->has_list && !is_permutation(src->list, H.A.n_rows)) { Y.src = -1; return; }
    std::vector<int> rows;
    build_waves(H.A, src->has_list ? src->list.data() : nullptr, H.A.n_rows, rows, W.ptr);
    if (W.ptr.size() - 1 > (size_t)H.A.n_rows / 8 + 64) {
        // (near-)sequential dependency chain, e.g. lexicographic GS on a banded operator: a
        // wave-major layout would scatter every row; keep the natural numbering + row lists
        Y = LevelLayout();
        return;
    }
    Y.order = rows;
    Y.pos.resize(rows.size());
    for (size_t i = 0; i < rows.size(); i++) Y.pos[(size_t)rows[i]] = (int)i;
    W.contiguous = true;
    W.nnz.assign(W.ptr.size() - 1, 0);
    for (size_t w = 0; w + 1 < W.ptr.size(); w++)
        for (long long k = W.ptr[w]; k < W.ptr[w + 1]; k++)
            W.nnz[w] += H.A.Ap[(size_t)rows[(size_t)k] + 1] - H.A.Ap[(size_t)rows[(size_t)k]];
}

// Permute level l's A / P / R into its layout Y (P's columns and R's rows into the next level's, `next`; null = they
// already are), build tiles, upload the operators and smoothers into levels[l]
int amgb_hierarchy::build_level(int l, const HostLevel &H, LevelLayout &Y, const LevelLayout *next)
{
    Level &L = levels[(size_t)l];
    L.has_pr = H.has_pr;
    const bool permuted = !Y.order.empty();
    const int *ord = permuted ? Y.order.data() : nullptr;
    const int *ps = permuted ? Y.pos.data() : nullptr;
    const int *psn = (next && !next->order.empty()) ? next->pos.data() : nullptr;
    const int *ordn = (next && !next->order.empty()) ? next->order.data() : nullptr;
    HostCsr Ap_;
    const HostCsr *Ause = &H.A;
    if (permuted) { permute_csr(H.A, ord, ps, Ap_); Ause = &Ap_; }
    WaveSchedule &W = Y.W;
    if (permuted) {
        RET(upload_csr(*Ause, L.A, &W.ptr, &W.tile_ptr, 0, 0, nullptr, S.use_value_codes));
        if (!S.use_tiles) W.tile_ptr.clear();
    } else {
        RET(upload_csr(*Ause, L.A, nullptr, nullptr, 0, 0, nullptr, S.use_value_codes));
    }
    if (H.has_pr) {
        HostCsr T;
        if (ord || psn) permute_csr(H.P, ord, psn, T);
        RET(upload_csr((ord || psn) ? T : H.P, L.P, nullptr, nullptr, 1, l, nullptr, S.use_value_codes));
        if (ordn || ps) permute_csr(H.R, ordn, ps, T);
        RET(upload_csr((ordn || ps) ? T : H.R, L.R, nullptr, nullptr, 2, l, nullptr, S.use_value_codes));
        const std::vector<int> *pv = permuted ? &Y.pos : nullptr;
        const bool same_lists = H.pre.kind == AMGB_SM_GAUSS_SEIDEL && H.post.kind == AMGB_SM_GAUSS_SEIDEL &&
                                H.pre.has_list == H.post.has_list && H.pre.list == H.post.list;
        const WaveSchedule *sh_pre = (permuted && (Y.src == 0)) ? &W : nullptr;
        const WaveSchedule *sh_post = (permuted && (Y.src == 1 || same_lists)) ? &W : nullptr;
        if (H.pre.kind != AMGB_SM_GAUSS_SEIDEL) sh_pre = nullptr;
        if (H.post.kind != AMGB_SM_GAUSS_SEIDEL) sh_post = nullptr;
        if (Y.src >= 2) sh_pre = sh_post = nullptr;                 // (decided just below for the C|F layout)
        if (permuted && Y.src >= 2) {                               // C|F layout: smoothers with the layout's lists
            const SmootherSpec &ref = (Y.src == 2) ? H.pre : H.post;
            auto same_cf = [&](const SmootherSpec &q) {
                return (q.kind == AMGB_SM_CF_JACOBI || q.kind == AMGB_SM_FC_JACOBI) && q.list == ref.list && q.list2 == ref.list2;
            };
            sh_pre = same_cf(H.pre) ? &W : nullptr;
            sh_post = same_cf(H.post) ? &W : nullptr;
        }
        RET(make_smoother(H.pre, *Ause, pv, sh_pre, L.pre));
        RET(make_smoother(H.post, *Ause, pv, sh_post, L.post));
        // a coarse level's pre-smoother starts from x = 0 on the first visit after descend's fill
        if (l >= 1 && S.use_zero_start && sh_pre != nullptr && H.pre.kind == AMGB_SM_GAUSS_SEIDEL &&
            H.pre.sweep != AMGB_SWEEP_BACKWARD)
            RET(prepare_zero_start(*Ause, W, L));
    }
    if (!H.has_pr && coarse_relax) RET(make_smoother(coarse_spec, *Ause, nullptr, nullptr, coarse_sm));
    if (S.verbose) {     // how each operator's tiles stream
        auto kind = [](const DevCsr &M) {
            return M.rcodes ? "row8" : M.pairs ? "pair8" : M.codes ? "val8" : (M.tiles ? "fp64" : "rows");
        };
        auto table = [](const DevCsr &M) {
            return (long long)M.ndict * (M.pairs ? (long long)sizeof(PairCode) : M.codes ? 8ll : 0ll) +
                   (long long)M.npatterns * (long long)sizeof(RowPattern);
        };
        fprintf(stderr, "[amgb] level %d A: %s %d entries (%lld B table)", l, kind(L.A), L.A.ndict, table(L.A));
        if (L.A.rcodes) fprintf(stderr, ", %d row patterns", L.A.npatterns);
        if (H.has_pr)
            fprintf(stderr, ", P: %s %d (%lld B), R: %s %d (%lld B)", kind(L.P), L.P.ndict, table(L.P), kind(L.R),
                    L.R.ndict, table(L.R));
        if (L.zs.A.Ap != nullptr)
            fprintf(stderr, ", zero-start A: %s %d (%lld B)", kind(L.zs.A), L.zs.A.ndict, table(L.zs.A));
        fprintf(stderr, "\n");
    }
    if (l == 0 && permuted) {
        RET(upload(&order0, Y.order.data(), (long long)Y.order.size()));
        RET(upload(&pos0, Y.pos.data(), (long long)Y.pos.size()));
        RET(dalloc(&io_tmp, H.A.n_rows));
    }
    if (l == 0) {                       // what amgb_hierarchy_replace_level0 compares a new level 0's smoothers with
        spec0[0] = H.pre;
        spec0[1] = H.post;
        spec0[0].Dinv.clear();
        spec0[1].Dinv.clear();
    }
    return AMGB_OK;
}

// Decide the wave-major row permutation of every Gauss-Seidel level, permute A/P/R accordingly on the
// host, build tiles, upload everything.
int amgb_hierarchy::finalize_levels()
{
    const int nl = (int)host.size();
    std::vector<LevelLayout> layout((size_t)nl);
    for (int l = 0; l < nl; l++) plan_layout(host[(size_t)l], layout[(size_t)l]);
    levels.resize((size_t)nl);
    for (int l = 0; l < nl; l++) {
        RET(build_level(l, host[(size_t)l], layout[(size_t)l], l + 1 < nl ? &layout[(size_t)l + 1] : nullptr));
        host[(size_t)l] = HostLevel();  // release the host copy level by level
    }
    host.clear();
    host.shrink_to_fit();
    return AMGB_OK;
}

// ------------------------------------------------------------------------------------------
// C ABI (1): hierarchy
// ------------------------------------------------------------------------------------------
extern "C" int amgb_hierarchy_create(int device, amgb_hierarchy **out)
{
    if (out == nullptr) return fail(AMGB_EINVAL, "out is null");
    *out = nullptr;
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(AMGB_EINVAL, "no such CUDA device");
    CK(cudaSetDevice(device));
    std::unique_ptr<amgb_hierarchy> h(new amgb_hierarchy());
    RET(read_settings(device, h->S));
    h->device = device;
    *out = h.release();
    return AMGB_OK;
}

extern "C" void amgb_hierarchy_destroy(amgb_hierarchy *h)
{
    if (h == nullptr) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (int k = 0; k < 4; k++) {
        if (h->graph[k]) cudaGraphExecDestroy(h->graph[k]);
        if (h->graph_stop[k]) cudaGraphExecDestroy(h->graph_stop[k]);
    }
    for (ManyWidth &mw : h->many)
        for (cudaGraphExec_t g : mw.graph)
            if (g) cudaGraphExecDestroy(g);
    for (void *p : h->allocs) cudaFree(p);
    if (h->norm_host) cudaFreeHost(h->norm_host);
    for (cudaEvent_t e : h->io_event)
        if (e) cudaEventDestroy(e);
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

static int copy_smoother(const amgb_smoother *in, const HostCsr &A, SmootherSpec &s)
{
    s = SmootherSpec();
    if (in == nullptr || in->kind == AMGB_SM_NONE) return AMGB_OK;
    s.kind = in->kind;
    s.iterations = in->iterations;
    s.sweep = in->sweep;
    s.omega = in->omega;
    if (s.iterations < 0) return fail(AMGB_EINVAL, "smoother iterations < 0");
    switch (in->kind) {
    case AMGB_SM_JACOBI: return AMGB_OK;
    case AMGB_SM_GAUSS_SEIDEL:
        if (s.sweep < 0 || s.sweep > 2)
            return fail(AMGB_EINVAL, "valid sweep directions: \"forward\", \"backward\", and \"symmetric\"");
        if (in->indices != nullptr) {
            s.has_list = true;
            s.list.assign(in->indices, in->indices + in->n_indices);
            for (int v : s.list)
                if (v < 0 || v >= A.n_rows) return fail(AMGB_EINVAL, "gauss_seidel_indexed: row index out of range");
        }
        return AMGB_OK;
    case AMGB_SM_BLOCK_JACOBI:
        s.bs = in->blocksize;
        if (s.bs < 1 || s.bs > 8 || A.n_rows % s.bs)
            return fail(AMGB_ENOTIMPL, "block_jacobi: blocksize must be 1..8 and divide n");
        if (in->Dinv == nullptr) return fail(AMGB_EINVAL, "block_jacobi: Dinv required");
        s.Dinv.assign(in->Dinv, in->Dinv + (size_t)A.n_rows * s.bs);
        return AMGB_OK;
    case AMGB_SM_BLOCK_GAUSS_SEIDEL:
        if (s.sweep < 0 || s.sweep > 2)
            return fail(AMGB_EINVAL, "valid sweep directions: \"forward\", \"backward\", and \"symmetric\"");
        s.bs = in->blocksize;
        if (s.bs < 1 || s.bs > 8 || A.n_rows % s.bs)
            return fail(AMGB_ENOTIMPL, "block_gauss_seidel: blocksize must be 1..8 and divide n");
        if (in->Dinv == nullptr) return fail(AMGB_EINVAL, "block_gauss_seidel: Dinv required");
        s.Dinv.assign(in->Dinv, in->Dinv + (size_t)A.n_rows * s.bs);
        return AMGB_OK;
    case AMGB_SM_JACOBI_NE:
    case AMGB_SM_GAUSS_SEIDEL_NE:
    case AMGB_SM_GAUSS_SEIDEL_NR:
        if (s.sweep < 0 || s.sweep > 2)
            return fail(AMGB_EINVAL, "valid sweep directions: \"forward\", \"backward\", and \"symmetric\"");
        if (in->Dinv == nullptr) return fail(AMGB_EINVAL, "normal-equation smoother: Dinv (n-vector) required");
        s.Dinv.assign(in->Dinv, in->Dinv + (size_t)A.n_rows);
        return AMGB_OK;
    case AMGB_SM_SCHWARZ: {
        if (s.sweep < 0 || s.sweep > 2)
            return fail(AMGB_EINVAL, "valid sweep directions: 'forward', 'backward', and 'symmetric'");
        if (in->indices2 == nullptr || in->n_indices2 < 1 || (in->n_indices > 0 && in->indices == nullptr))
            return fail(AMGB_EINVAL, "schwarz: subdomain / subdomain_ptr required");
        s.list.assign(in->indices, in->indices + in->n_indices);
        s.list2.assign(in->indices2, in->indices2 + in->n_indices2);
        if (s.list2.front() != 0 || s.list2.back() != (int)s.list.size()) return fail(AMGB_EINVAL, "schwarz: subdomain_ptr inconsistent");
        long long tsize = 0;
        for (size_t k = 0; k + 1 < s.list2.size(); k++) {
            const long long m = s.list2[k + 1] - s.list2[k];
            if (m < 0) return fail(AMGB_EINVAL, "schwarz: subdomain_ptr not monotone");
            tsize += m * m;
        }
        for (int v : s.list)
            if (v < 0 || v >= A.n_rows) return fail(AMGB_EINVAL, "schwarz: row index out of range");
        {   // a row listed twice in ONE subdomain would be updated by two lanes at once
            std::vector<int> seen((size_t)A.n_rows, -1);
            for (size_t k = 0; k + 1 < s.list2.size(); k++)
                for (int q = s.list2[k]; q < s.list2[k + 1]; q++) {
                    if (seen[(size_t)s.list[(size_t)q]] == (int)k) return fail(AMGB_ENOTIMPL, "schwarz: a subdomain lists a row twice");
                    seen[(size_t)s.list[(size_t)q]] = (int)k;
                }
        }
        if (in->Dinv == nullptr && tsize > 0) return fail(AMGB_EINVAL, "schwarz: inv_subblock required");
        s.Dinv.assign(in->Dinv, in->Dinv + tsize);
        return AMGB_OK;
    }
    case AMGB_SM_CF_BLOCK_JACOBI:
    case AMGB_SM_FC_BLOCK_JACOBI: {
        s.bs = in->blocksize;
        if (s.bs < 1 || s.bs > 8 || A.n_rows % s.bs)
            return fail(AMGB_ENOTIMPL, "cf_block_jacobi: blocksize must be 1..8 and divide n");
        if (in->Dinv == nullptr) return fail(AMGB_EINVAL, "cf_block_jacobi: Dinv required");
        if (in->n_indices < 0 || in->n_indices2 < 0 || (in->n_indices > 0 && in->indices == nullptr) ||
            (in->n_indices2 > 0 && in->indices2 == nullptr))
            return fail(AMGB_EINVAL, "cf_block_jacobi: null block-row list");
        s.Dinv.assign(in->Dinv, in->Dinv + (size_t)A.n_rows * s.bs);
        s.list.assign(in->indices, in->indices + in->n_indices);
        s.list2.assign(in->indices2, in->indices2 + in->n_indices2);
        s.f_iterations = in->f_iterations;
        s.c_iterations = in->c_iterations;
        if (s.f_iterations < 0 || s.c_iterations < 0) return fail(AMGB_EINVAL, "cf_block_jacobi: iterations < 0");
        const int nb = A.n_rows / s.bs;
        for (int v : s.list)
            if (v < 0 || v >= nb) return fail(AMGB_EINVAL, "cf_block_jacobi: block-row index out of range");
        for (int v : s.list2)
            if (v < 0 || v >= nb) return fail(AMGB_EINVAL, "cf_block_jacobi: block-row index out of range");
        return AMGB_OK;
    }
    case AMGB_SM_POLYNOMIAL:
        if (in->coefficients == nullptr || in->n_coefficients < 1)
            return fail(AMGB_EINVAL, "polynomial: at least one coefficient required");
        s.coef.assign(in->coefficients, in->coefficients + in->n_coefficients);
        return AMGB_OK;
    case AMGB_SM_JACOBI_INDEXED:
    case AMGB_SM_CF_JACOBI:
    case AMGB_SM_FC_JACOBI:
        if (in->n_indices < 0 || in->n_indices2 < 0 || (in->n_indices > 0 && in->indices == nullptr) ||
            (in->n_indices2 > 0 && in->indices2 == nullptr))
            return fail(AMGB_EINVAL, "indexed Jacobi: null row list");
        s.list.assign(in->indices, in->indices + in->n_indices);
        if (in->kind != AMGB_SM_JACOBI_INDEXED) {
            s.list2.assign(in->indices2, in->indices2 + in->n_indices2);
            s.f_iterations = in->f_iterations;
            s.c_iterations = in->c_iterations;
            if (s.f_iterations < 0 || s.c_iterations < 0) return fail(AMGB_EINVAL, "CF Jacobi: iterations < 0");
        }
        for (int v : s.list)
            if (v < 0 || v >= A.n_rows) return fail(AMGB_EINVAL, "indexed Jacobi: row index out of range");
        for (int v : s.list2)
            if (v < 0 || v >= A.n_rows) return fail(AMGB_EINVAL, "indexed Jacobi: row index out of range");
        return AMGB_OK;
    }
    return fail(AMGB_ENOTIMPL, "smoother kind outside the hot-path scope");
}

extern "C" int amgb_hierarchy_add_level(amgb_hierarchy *h, const amgb_matrix *A, const amgb_matrix *P,
                                        const amgb_matrix *R, const amgb_smoother *pre,
                                        const amgb_smoother *post)
{
    if (h == nullptr) return fail(AMGB_EINVAL, "null hierarchy");
    if (h->finalized) return fail(AMGB_ESTATE, "hierarchy already finalized");
    if (!h->host.empty() && !h->host.back().has_pr)
        return fail(AMGB_ESTATE, "previous level was added as the coarsest (no P/R)");
    h->host.emplace_back();
    HostLevel &L = h->host.back();
    int rc = to_host_csr(A, L.A, "A");
    if (rc == AMGB_OK && L.A.n_rows != L.A.n_cols) rc = fail(AMGB_EINVAL, "expected square matrix");   // relaxation.py:81-82
    if (rc == AMGB_OK && h->host.size() > 1 && h->host[h->host.size() - 2].P.n_cols != L.A.n_rows)
        rc = fail(AMGB_EINVAL, "level size does not match the previous level's P");
    if (rc == AMGB_OK && (P == nullptr) != (R == nullptr)) rc = fail(AMGB_EINVAL, "P and R must be given together");
    if (rc == AMGB_OK && P != nullptr) {
        rc = to_host_csr(P, L.P, "P");
        if (rc == AMGB_OK) rc = to_host_csr(R, L.R, "R");
        if (rc == AMGB_OK && (L.P.n_rows != L.A.n_rows || L.R.n_cols != L.A.n_rows || L.R.n_rows != L.P.n_cols))
            rc = fail(AMGB_EINVAL, "P/R shapes inconsistent with A");
        L.has_pr = true;
        if (rc == AMGB_OK) rc = copy_smoother(pre, L.A, L.pre);
        if (rc == AMGB_OK) rc = copy_smoother(post, L.A, L.post);
    }
    if (rc != AMGB_OK) h->host.pop_back();
    return rc;
}

extern "C" int amgb_hierarchy_set_coarse_pinv(amgb_hierarchy *h, int32_t n, const double *pinv,
                                              int32_t coarse_is_zero)
{
    if (h == nullptr) return fail(AMGB_EINVAL, "null hierarchy");
    if (h->finalized) return fail(AMGB_ESTATE, "hierarchy already finalized");
    if (h->host.empty()) return fail(AMGB_ESTATE, "no levels");
    if (n != h->host.back().A.n_rows) return fail(AMGB_EINVAL, "pinv size != coarsest level size");
    h->coarse_zero = coarse_is_zero != 0;
    h->coarse_n = n;
    if (!h->coarse_zero) {
        if (pinv == nullptr) return fail(AMGB_EINVAL, "pinv is null");
        h->coarse_host.assign(pinv, pinv + (size_t)n * n);
    }
    h->have_coarse = true;
    return AMGB_OK;
}

extern "C" int amgb_hierarchy_set_coarse_relaxation(amgb_hierarchy *h, const amgb_smoother *sm)
{
    if (h == nullptr || sm == nullptr) return fail(AMGB_EINVAL, "null argument");
    if (h->finalized) return fail(AMGB_ESTATE, "hierarchy already finalized");
    if (h->host.empty()) return fail(AMGB_ESTATE, "no levels");
    if (h->host.back().has_pr) return fail(AMGB_ESTATE, "the coarsest level must be added first (without P/R)");
    if (sm->kind == AMGB_SM_NONE) return fail(AMGB_EINVAL, "coarse relaxation: a smoother kind is required");
    RET(copy_smoother(sm, h->host.back().A, h->coarse_spec));
    h->coarse_relax = true;
    h->coarse_zero = false;
    h->coarse_n = h->host.back().A.n_rows;
    h->have_coarse = true;
    return AMGB_OK;
}

extern "C" int amgb_hierarchy_finalize(amgb_hierarchy *h, void *stream)
{
    if (h == nullptr) return fail(AMGB_EINVAL, "null hierarchy");
    if (h->finalized) return fail(AMGB_ESTATE, "already finalized");
    if (h->host.empty()) return fail(AMGB_ESTATE, "no levels");
    if (h->host.back().has_pr) return fail(AMGB_ESTATE, "last level must be added without P/R");
    if (!h->have_coarse) return fail(AMGB_ESTATE, "coarse solver not set");
    CK(cudaSetDevice(h->device));
    const Settings &S = h->S;
    if (stream != nullptr) {
        h->stream = (cudaStream_t)stream;
    } else {
        CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        h->own_stream = true;
    }
    RET(h->finalize_levels());
    for (Level &L : h->levels) {
        if (!L.has_pr) continue;
        RET(h->resident_prepare(L, L.pre));
        RET(h->resident_prepare(L, L.post));
    }
    {   // coarse tail: the deepest run of levels whose operators are all small and block-smoother free
        const int nl = (int)h->levels.size();
        int tl = nl;
        for (int l = nl - 1; l >= 1; l--) {
            const Level &L = h->levels[(size_t)l];
            // only the kinds the cluster interpreter knows (none, Jacobi, Gauss-Seidel) may run in the tail
            const bool blocky = L.has_pr && (L.pre.kind > AMGB_SM_GAUSS_SEIDEL || L.post.kind > AMGB_SM_GAUSS_SEIDEL);
            const bool coarse_blocky = !L.has_pr && h->coarse_relax && h->coarse_sm.kind > AMGB_SM_GAUSS_SEIDEL;
            if (L.A.nnz > S.tail_nnz_limit || blocky || coarse_blocky) break;
            tl = l;
        }
        if (tl < nl && S.tail_grid) {
            // one CTA per SM, all co-resident (cooperative launch): never more CTAs than the device can hold at once
            int per_sm = 0;
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, coarse_grid_kernel, kGridThreads, 0));
            if (per_sm < 1) return fail(AMGB_ECUDA, "coarse_grid_kernel does not fit an SM");
            RET(h->dalloc(&h->grid_sync, 1));
            CK(cudaMemset(h->grid_sync, 0, sizeof(GridSync)));
            h->tail_level = tl;
        } else if (tl < nl) {
            CK(cudaFuncSetAttribute(tail_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
            h->tail_csize = 1;
            for (int c = 16; c >= 1; c >>= 1) {
                if (c > S.tail_cluster) continue;
                cudaLaunchConfig_t cfg = {};
                cfg.gridDim = dim3((unsigned)c); cfg.blockDim = dim3(kTailThreads);
                cudaLaunchAttribute at[1];
                at[0].id = cudaLaunchAttributeClusterDimension;
                at[0].val.clusterDim.x = (unsigned)c; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
                cfg.attrs = at; cfg.numAttrs = 1;
                int nclusters = 0;
                if (cudaOccupancyMaxActiveClusters(&nclusters, tail_kernel, &cfg) == cudaSuccess && nclusters >= 1) {
                    h->tail_csize = c;
                    break;
                }
                cudaGetLastError();
            }
            h->tail_level = tl;
        }
        if (S.verbose)
            fprintf(stderr, "[amgb] levels=%d tail_level=%d cluster=%d tile_cfg=%d ctas/sm=%d hints=%d\n", nl,
                    h->tail_level < nl ? h->tail_level : -1, h->tail_csize, S.tile_cfg, S.tile_ctas[OP_GS], S.tile_hints);
    }
    if (!h->coarse_zero && !h->coarse_relax)
        RET(h->upload(&h->coarse_pinv, h->coarse_host.data(), (long long)h->coarse_host.size()));
    h->coarse_host.clear();
    for (Level &L : h->levels) {
        const long long n = L.A.n_rows;
        RET(h->dalloc(&L.x_home, n + 2));      // +2: the TMA reads whole 16-byte groups
        RET(h->dalloc(&L.xalt, n + 2));
        RET(h->dalloc(&L.b, n + 2));
        RET(h->dalloc(&L.r, n + 2));
        L.x = L.x_home;
        if ((L.has_pr && (L.pre.kind == AMGB_SM_POLYNOMIAL || L.post.kind == AMGB_SM_POLYNOMIAL)) ||
            (!L.has_pr && h->coarse_relax && h->coarse_sm.kind == AMGB_SM_POLYNOMIAL)) {
            RET(h->dalloc(&L.poly[0], n + 2));
            RET(h->dalloc(&L.poly[1], n + 2));
        }
    }
    // x 3: the stop test's residual may be a Gauss-Seidel wave's partials and two residual launches' (smooth_residual)
    h->n_partials = std::max<long long>(3 * h->partials_len(h->levels[0].A), 1);
    RET(h->dalloc(&h->partials, h->n_partials));
    RET(h->ensure_norms(128));
    RET(h->dalloc(&h->sumsq_parts, kSumsqBlocks));
    CK(cudaHostAlloc((void **)&h->norm_host, sizeof(double) * 2, cudaHostAllocDefault));
    h->finalized = true;
    return AMGB_OK;
}

extern "C" int amgb_hierarchy_num_levels(const amgb_hierarchy *h)
{
    return h ? (int)(h->finalized ? h->levels.size() : h->host.size()) : 0;
}
extern "C" int64_t amgb_hierarchy_device_bytes(const amgb_hierarchy *h) { return h ? h->dev_bytes : 0; }
extern "C" int64_t amgb_hierarchy_last_launches(const amgb_hierarchy *h) { return h ? h->last_launches : 0; }

extern "C" int amgb_host_alloc(size_t bytes, void **out)
{
    if (out == nullptr) return fail(AMGB_EINVAL, "out is null");
    CK(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
    return AMGB_OK;
}
extern "C" int amgb_host_free(void *p)
{
    if (p) CK(cudaFreeHost(p));
    return AMGB_OK;
}

static int check_cycle_args(amgb_hierarchy *h, int32_t cycle, int32_t cpl)
{
    if (h == nullptr) return fail(AMGB_EINVAL, "null hierarchy");
    if (!h->finalized) return fail(AMGB_ESTATE, "hierarchy not finalized");
    if (cycle < 0 || cycle > AMGB_CYCLE_AMLI) return fail(AMGB_EINVAL, "Unrecognized cycle type");
    if (cpl < 0) return fail(AMGB_EINVAL, "cycles_per_level < 0");
    return AMGB_OK;
}

extern "C" int amgb_hierarchy_set_io_stream(amgb_hierarchy *h, void *stream)
{
    if (h == nullptr) return fail(AMGB_EINVAL, "null hierarchy");
    h->io_stream = (cudaStream_t)stream;
    return AMGB_OK;
}

// p is device (or managed) memory on `device`.  The emulator (tests/emu) knows no pointer attributes: there device
// memory is whatever lies inside one of its allocations.
static bool is_device_memory(const void *p, int device)
{
#ifdef AMGB_EMU
    (void)device;
    const uintptr_t a = (uintptr_t)p;
    auto it = emu::g.allocs.upper_bound(a);
    if (it == emu::g.allocs.begin()) return false;
    --it;
    return a < it->first + it->second;
#else
    cudaPointerAttributes attr = {};
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) && attr.device == device;
#endif
}

// work enqueued on `waiter` from now on follows the work enqueued on `signaller` so far (one event, created on first
// use).  The emulator completes every operation before the call that issues it returns: nothing to order there.
static int stream_wait(cudaStream_t waiter, cudaStream_t signaller, cudaEvent_t &ev)
{
#ifdef AMGB_EMU
    (void)waiter; (void)signaller; (void)ev;
#else
    if (ev == nullptr) CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CK(cudaEventRecord(ev, signaller));
    CK(cudaStreamWaitEvent(waiter, ev, 0));
#endif
    return AMGB_OK;
}

// The caller's vectors of one solve call.  Without AMGB_FLAG_DEVICE_IO they are host arrays, staged by the copy-in /
// copy-out helpers.  With it they are device memory on the hierarchy's device, checked before anything is enqueued;
// the engine's stream then waits for the caller's stream (io_stream) on entry, and io_stream waits for the engine's
// stream on exit -- also when the call fails half way, so that the caller never races work still in flight.
struct CallerIo {
    amgb_hierarchy *h;
    const bool dev;
    bool ordered = false;          // the engine's stream waits on io_stream: io_stream must wait on it in turn

    CallerIo(amgb_hierarchy *h_, int32_t flags) : h(h_), dev((flags & AMGB_FLAG_DEVICE_IO) != 0) {}
    ~CallerIo() { end(); }
    CallerIo(const CallerIo &) = delete;
    CallerIo &operator=(const CallerIo &) = delete;

    // after cudaSetDevice(h->device)
    int begin(const void *in, const void *out)
    {
        if (!dev) return AMGB_OK;
        for (const void *p : {in, out})
            if (!is_device_memory(p, h->device))
                return fail(AMGB_EINVAL, "AMGB_FLAG_DEVICE_IO: a vector is not device memory on the hierarchy's device");
        if (h->io_stream == nullptr || h->io_stream == h->stream) return AMGB_OK;
        RET(stream_wait(h->stream, h->io_stream, h->io_event[0]));
        ordered = true;
        return AMGB_OK;
    }
    int end()
    {
        if (!ordered) return AMGB_OK;
        ordered = false;
        return stream_wait(h->io_stream, h->stream, h->io_event[1]);
    }
    cudaMemcpyKind in_kind() const { return dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice; }
    cudaMemcpyKind out_kind() const { return dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost; }
};

// bring b / x0 into the level-0 buffers (wave-major order if level 0 is permuted).  Host arrays are staged through
// io_tmp; device arrays (kind == cudaMemcpyDeviceToDevice) are gathered straight from the caller's memory.
static int load_level0(amgb_hierarchy *h, const double *b, const double *x, cudaMemcpyKind kind)
{
    Level &L0 = h->levels[0];
    const size_t bytes = sizeof(double) * (size_t)L0.A.n_rows;
    cudaStream_t s = h->stream;
    L0.x = L0.x_home;
    if (h->order0 == nullptr) {
        CK(cudaMemcpyAsync(L0.b, b, bytes, kind, s));
        if (x == nullptr) return h->launch_count_fill(L0.x, L0.A.n_rows);
        CK(cudaMemcpyAsync(L0.x, x, bytes, kind, s));
        return AMGB_OK;
    }
    const bool dev = kind == cudaMemcpyDeviceToDevice;
    if (!dev) CK(cudaMemcpyAsync(h->io_tmp, b, bytes, kind, s));
    RET(h->gather(dev ? b : h->io_tmp, h->order0, L0.b, L0.A.n_rows));
    if (x == nullptr) return h->launch_count_fill(L0.x, L0.A.n_rows);   // x0 = 0: nothing to copy
    if (!dev) CK(cudaMemcpyAsync(h->io_tmp, x, bytes, kind, s));
    RET(h->gather(dev ? x : h->io_tmp, h->order0, L0.x, L0.A.n_rows));
    return AMGB_OK;
}

// the level-0 iterate -> x in the caller's numbering (a device x, kind == cudaMemcpyDeviceToDevice, is scattered into
// directly)
static int store_level0(amgb_hierarchy *h, double *x, cudaMemcpyKind kind)
{
    Level &L0 = h->levels[0];
    const size_t bytes = sizeof(double) * (size_t)L0.A.n_rows;
    if (h->order0 == nullptr) {
        CK(cudaMemcpyAsync(x, L0.x, bytes, kind, h->stream));
        return AMGB_OK;
    }
    if (kind == cudaMemcpyDeviceToDevice) return h->gather(L0.x, h->pos0, x, L0.A.n_rows);
    RET(h->gather(L0.x, h->pos0, h->io_tmp, L0.A.n_rows));
    CK(cudaMemcpyAsync(x, h->io_tmp, bytes, kind, h->stream));
    return AMGB_OK;
}

extern "C" int amgb_solve_ex(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t maxiter,
                             int32_t cycle, int32_t cycles_per_level, int32_t flags, double *residuals,
                             int32_t *n_residuals, int32_t *info);

extern "C" int amgb_solve(amgb_hierarchy *h, const double *b_host, double *x_host, double tol,
                          int32_t maxiter, int32_t cycle, int32_t cycles_per_level, double *residuals,
                          int32_t *n_residuals, int32_t *info)
{
    return amgb_solve_ex(h, b_host, x_host, tol, maxiter, cycle, cycles_per_level, 0, residuals, n_residuals, info);
}

extern "C" int amgb_solve_ex(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t maxiter,
                             int32_t cycle, int32_t cycles_per_level, int32_t flags, double *residuals,
                             int32_t *n_residuals, int32_t *info)
{
    RET(check_cycle_args(h, cycle, cycles_per_level));
    if (b_host == nullptr || x_host == nullptr) return fail(AMGB_EINVAL, "null host vector");
    if (maxiter < 1) return fail(AMGB_EINVAL, "maxiter must be >= 1");
    CK(cudaSetDevice(h->device));
    CallerIo io(h, flags);
    RET(io.begin(b_host, x_host));
    Level &L0 = h->levels[0];
    cudaStream_t s = h->stream;
    h->launches = 0;
    RET(h->ensure_norms(maxiter + 1));
    RET(load_level0(h, b_host, (flags & AMGB_FLAG_X0_ZERO) ? nullptr : x_host, io.in_kind()));

    // normb (multilevel.py:540-542) is only needed by the stop test; reduce it on the device
    double normb = 1.0;
    if (tol > 0.0) {
        sumsq_partials_kernel<<<sumsq_blocks(h->S), 256, 0, s>>>(L0.b, L0.A.n_rows, h->sumsq_parts);
        CK(cudaGetLastError());
        reduce_partials_kernel<<<1, 1024, 0, s>>>(h->sumsq_parts, sumsq_blocks(h->S), h->norms2);
        CK(cudaGetLastError());
        h->launches += 2;
        CK(cudaMemcpyAsync(h->norm_host, h->norms2, sizeof(double), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        normb = std::sqrt(h->norm_host[0]);
        if (normb == 0.0) normb = 1.0;
    }
    if (flags & AMGB_FLAG_X0_ZERO) {
        // x0 = 0: the initial residual b - A 0 is b itself (:545) -- one pass over b instead of one over A
        sumsq_partials_kernel<<<sumsq_blocks(h->S), 256, 0, s>>>(L0.b, L0.A.n_rows, h->sumsq_parts);
        CK(cudaGetLastError());
        reduce_partials_kernel<<<1, 1024, 0, s>>>(h->sumsq_parts, sumsq_blocks(h->S), h->norms2);
        CK(cudaGetLastError());
        h->launches += 2;
    } else {
        RET(h->residual_norm2(0));                                 // :545
    }
    int it = 0, conv = -1;
    while (true) {
        it++;
        RET(h->iteration_norm2(cycle, cycles_per_level, it));      // :559-563, :567
        if (tol > 0.0) {
            CK(cudaMemcpyAsync(h->norm_host, h->norms2 + it, sizeof(double), cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            if (std::sqrt(h->norm_host[0]) < tol * normb) { conv = 0; break; }   // :574
        }
        if (it == maxiter) { conv = it; break; }                  // :579
    }
    RET(store_level0(h, x_host, io.out_kind()));
    RET(io.end());
    if (!io.dev || residuals != nullptr) {     // device I/O without a residual list: nothing to wait for
        std::vector<double> n2((size_t)it + 1);
        CK(cudaMemcpyAsync(n2.data(), h->norms2, sizeof(double) * ((size_t)it + 1), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        if (residuals != nullptr)
            for (int k = 0; k <= it; k++) residuals[k] = std::sqrt(n2[(size_t)k]);
    }
    if (n_residuals != nullptr) *n_residuals = it + 1;
    if (info != nullptr) *info = conv;
    h->last_launches = h->launches;
    return AMGB_OK;
}

extern "C" int amgb_solve_device(amgb_hierarchy *h, const double *b_dev, double *x_dev, int32_t ncycles,
                                 int32_t cycle, int32_t cycles_per_level, double *norms2_dev)
{
    RET(check_cycle_args(h, cycle, cycles_per_level));
    if (b_dev == nullptr || x_dev == nullptr) return fail(AMGB_EINVAL, "null device vector");
    if (ncycles < 0) return fail(AMGB_EINVAL, "ncycles < 0");
    CK(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    h->launches = 0;
    RET(load_level0(h, b_dev, x_dev, cudaMemcpyDeviceToDevice));
    if (norms2_dev != nullptr) {
        RET(h->ensure_norms(ncycles + 1));
        RET(h->residual_norm2(0));
    }
    for (int it = 1; it <= ncycles; it++) {
        if (norms2_dev != nullptr) RET(h->iteration_norm2(cycle, cycles_per_level, it));
        else RET(h->one_iteration(cycle, cycles_per_level));
    }
    RET(store_level0(h, x_dev, cudaMemcpyDeviceToDevice));
    if (norms2_dev != nullptr)
        CK(cudaMemcpyAsync(norms2_dev, h->norms2, sizeof(double) * ((size_t)ncycles + 1),
                           cudaMemcpyDeviceToDevice, s));
    h->last_launches = h->launches;
    return AMGB_OK;
}

#include "abi_krylov.cuh"      // amgb_solve_cg, amgb_solve_gmres (Householder, flexible, modified Gram-Schmidt)
#include "abi_many.cuh"        // amgb_solve_many: up to eight right-hand sides per pass over the hierarchy
#include "abi_many_krylov.cuh" // amgb_solve_many_cg / _bicgstab: batched preconditioned CG and BiCGStab
#include "abi_many_gmres.cuh"  // amgb_solve_many_gmres: batched Householder, flexible and modified Gram-Schmidt GMRES
#include "abi_krylov_more.cuh"      // amgb_solve_krylov: CGNR, CGNE, minimal residual, steepest descent
#include "abi_many_krylov_more.cuh" // amgb_solve_many_krylov: the same four on up to eight right-hand sides
#include "abi_replace.cuh"     // amgb_hierarchy_replace_level0: a new fine-level matrix under a resident hierarchy

// One un-graphed cycle with a CUDA-event pair around every operator launch of the cycle.
// rec[k*6 + {0..5}] = level, op (0 spmv/R, 1 residual, 2 prolong+add, 3 jacobi, 4 gs wave, 5 block jacobi,
// 6 = the whole coarse tail as one cluster kernel: rows = #steps, 12 = a sweep's last Gauss-Seidel wave that also
// writes its rows' residual),
// rows, nnz, algorithmic bytes, milliseconds.  Returns the number of records (<= max_records).
extern "C" int amgb_profile_cycle(amgb_hierarchy *h, int32_t cycle, double *rec, int32_t max_records,
                                  int32_t *n_records)
{
    RET(check_cycle_args(h, cycle, 1));
    if (rec == nullptr || n_records == nullptr) return fail(AMGB_EINVAL, "null output");
    if (h->levels.size() < 2) { *n_records = 0; return AMGB_OK; }
    CK(cudaSetDevice(h->device));
    h->prof.clear();
    RET(h->prepare_tail(cycle, 1));
    h->profiling = true;
    int rc = h->cycle(0, cycle, 1);
    h->profiling = false;
    cudaError_t e = cudaStreamSynchronize(h->stream);
    int n = 0;
    for (ProfRec &r : h->prof) {
        float ms = 0.f;
        if (rc == AMGB_OK && e == cudaSuccess && cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess && n < max_records) {
            double *o = rec + (size_t)n * 6;
            o[0] = r.level; o[1] = r.op; o[2] = (double)r.rows; o[3] = (double)r.nnz; o[4] = r.bytes; o[5] = ms;
            n++;
        }
        cudaEventDestroy(r.e0);
        cudaEventDestroy(r.e1);
    }
    h->prof.clear();
    *n_records = n;
    if (rc != AMGB_OK) return rc;
    if (e != cudaSuccess) return fail(AMGB_ECUDA, std::string("profile sync: ") + cudaGetErrorString(e));
    return AMGB_OK;
}

#include "abi_operator.cuh"    // amgb_operator_*, amgb_arnoldi_*, amgb_debug_*, amgb_dev_*
#include "abi_host.cuh"        // amgb_host_*, amgb_host_relax, amgb_host_csr_matmat
#include "abi_comm.cuh"        // amgb_comm_*: halo exchange over NVLink peer memory (multi-GPU)
