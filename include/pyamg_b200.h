/*
 * pyamg_b200.h -- C ABI of the H100-native AMG solve-phase engine (libpyamg_b200.so).
 *
 * This is the drop-in boundary for pyamg's solve phase (SURVEY.md 8(b)).  Plain pointers and
 * sizes only; no torch / numpy / C++ types cross it.  Three groups of entry points:
 *
 *  (1) amgb_hierarchy_* / amgb_solve / amgb_cycle -- replaces MultilevelSolver.solve and the
 *      recursive cycle driver MultilevelSolver.__solve (pyamg/multilevel.py:398-582, :584-662).
 *      The hierarchy (A_k, P_k, R_k as CSR/BSR host arrays, smoother descriptors, the dense
 *      coarse pseudo-inverse) is uploaded ONCE to HBM; every solve() then takes HOST b/x0 and
 *      returns HOST x, exactly like the reference's NumPy-in / NumPy-out call -- or, with
 *      AMGB_FLAG_DEVICE_IO, reads and writes the caller's DEVICE vectors in place.
 *  (2) amgb_host_* -- same argument lists as the reference's pybind11 FFI for its native sweeps
 *      (pyamg/amg_core/relaxation_bind.cpp: jacobi :847-854, bsr_jacobi, gauss_seidel,
 *      gauss_seidel_indexed, block_jacobi <- relaxation.h:309-346, :472-562, :48-76, :736-768,
 *      :1021-1090): HOST arrays in, x updated in place.  Each array parameter is followed by
 *      its length, as the reference's binding generator emits them (bindthem.py:74-81).
 *  (3) amgb_dev_* -- the individual sm_90a kernels on DEVICE pointers + a CUDA stream, for
 *      callers that keep vectors resident (Krylov accelerators, the multi-GPU layer, tests).
 *
 * All values are fp64, all indices int32 (the reference's only index instantiation,
 * pyamg/amg_core/instantiate.yml:2-6).  Every function returns 0 on success and a negative
 * AMGB_E* code on failure; amgb_last_error() gives the message (thread-local).  Nothing here
 * ever falls back to a CPU implementation: without a CUDA device every call fails.
 */
#ifndef PYAMG_B200_H
#define PYAMG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AMGB_OK 0
#define AMGB_EINVAL (-1)      /* bad argument (maps to ValueError/TypeError in the Python mirror) */
#define AMGB_ECUDA (-2)       /* CUDA runtime / NCCL failure */
#define AMGB_ENOTIMPL (-3)    /* smoother / format outside the hot-path scope (NotImplementedError) */
#define AMGB_ESTATE (-4)      /* call order violated (e.g. solve before finalize) */

/* smoother kinds (what lvl.presmoother / lvl.postsmoother resolve to; SURVEY.md descriptor table) */
#define AMGB_SM_NONE 0
#define AMGB_SM_JACOBI 1          /* relaxation.jacobi        (CSR, or BSR viewed point-wise)   */
#define AMGB_SM_GAUSS_SEIDEL 2    /* relaxation.gauss_seidel / gauss_seidel_indexed: a row list
                                     executed in dependency waves == the sequential sweep       */
#define AMGB_SM_BLOCK_JACOBI 3    /* relaxation.block_jacobi  (BSR + Dinv)                       */
/* SURVEY.md 8(f)-2: the cheap smoothers that share the SpMV / row-sweep core */
#define AMGB_SM_POLYNOMIAL 4      /* relaxation.polynomial (relaxation.py:585-659): x += p(A)(b - A x), Horner;
                                     what 'chebyshev' and 'richardson' resolve to (smoothing.py:611-647)      */
#define AMGB_SM_JACOBI_INDEXED 5  /* relaxation.jacobi_indexed (relaxation.py:1081-1138 -> relaxation.h:382-427) */
#define AMGB_SM_CF_JACOBI 6       /* relaxation.cf_jacobi (relaxation.py:1141-1203): C sweeps, then F sweeps     */
#define AMGB_SM_FC_JACOBI 7       /* relaxation.fc_jacobi (relaxation.py:1206-1268): F sweeps, then C sweeps     */
#define AMGB_SM_BLOCK_GAUSS_SEIDEL 8  /* relaxation.block_gauss_seidel (relaxation.py:502-582 ->
                                     relaxation.h:1242-1298): block rows in dependency waves == the sequential sweep */
#define AMGB_SM_CF_BLOCK_JACOBI 9 /* relaxation.cf_block_jacobi (relaxation.py:1271-1339 -> block_jacobi_indexed,
                                     relaxation.h:1113-1172): indices / indices2 list BLOCK rows (C / F), Dinv as for
                                     block Jacobi; AIR's smoother for block systems */
#define AMGB_SM_FC_BLOCK_JACOBI 10 /* relaxation.fc_block_jacobi (relaxation.py:1342-1412) */
/* normal-equation smoothers (Kaczmarz family): the descriptor's Dinv is an n-vector -- 1 / diag(A A^H) for the NE
 * kinds, 1 / diag(A^H A) for NR (util.get_diagonal(norm_eq = 2 | 1), relaxation.py:798, :881, :969); the engine
 * keeps its own column-sorted copies of A and A^T for them (the reference sorts the operator in place there) */
#define AMGB_SM_JACOBI_NE 11        /* relaxation.jacobi_ne (relaxation.py:734-812 -> relaxation.h:579-606) */
#define AMGB_SM_GAUSS_SEIDEL_NE 12  /* relaxation.gauss_seidel_ne (relaxation.py:815-901 -> relaxation.h:633-657):
                                       row projections in dependency waves of the A A^T conflict graph */
#define AMGB_SM_GAUSS_SEIDEL_NR 13  /* relaxation.gauss_seidel_nr (relaxation.py:904-999 -> relaxation.h:684-713):
                                       column projections on the residual, waves of the A^T A conflict graph */
#define AMGB_SM_SCHWARZ 14          /* relaxation.schwarz (relaxation.py:157-262 -> overlapping_schwarz_csr,
                                       relaxation.h:818-880): multiplicative overlapping Schwarz.  indices = the
                                       subdomains' row lists back to back, indices2 = their n_sub + 1 offsets, Dinv =
                                       the (pseudo-)inverses of the subdomain blocks, row-major, back to back */

#define AMGB_SWEEP_FORWARD 0
#define AMGB_SWEEP_BACKWARD 1
#define AMGB_SWEEP_SYMMETRIC 2

#define AMGB_CYCLE_V 0
#define AMGB_CYCLE_W 1
#define AMGB_CYCLE_F 2
#define AMGB_CYCLE_AMLI 3   /* multilevel.py:631-657 (two A_c-orthogonalised coarse corrections per level) */

typedef struct amgb_hierarchy amgb_hierarchy;

/* A sparse operator in HOST memory. block_r == block_c == 1 means CSR; otherwise BSR with
 * row-major block_r x block_c blocks (scipy bsr_array.data layout).  n_rows/n_cols are POINT
 * dimensions. indptr has n_rows/block_r + 1 entries. */
typedef struct {
    int32_t n_rows, n_cols;
    int32_t block_r, block_c;
    int64_t nnz_blocks;           /* len(indices) */
    const int32_t *indptr;
    const int32_t *indices;
    const double *data;           /* nnz_blocks * block_r * block_c values */
} amgb_matrix;

/* One smoother application (pre or post) on a level. */
typedef struct {
    int32_t kind;                 /* AMGB_SM_* */
    int32_t iterations;
    int32_t sweep;                /* AMGB_SWEEP_* (Gauss-Seidel only) */
    int32_t blocksize;            /* block Jacobi only */
    double omega;                 /* Jacobi / block Jacobi: already divided by rho (smoothing.py:501-508);
                                     Gauss-Seidel: SOR factor (forward/backward only, relaxation.py:326-338) */
    const int32_t *indices;       /* Gauss-Seidel: explicit row list (gauss_seidel_indexed), or NULL
                                     for the natural order 0..n-1 (gauss_seidel) */
    int64_t n_indices;
    const double *Dinv;           /* block Jacobi / block Gauss-Seidel: (n/bs, bs, bs) row-major block-diagonal inverses */
    /* ---- fields below exist since amgb_version() >= 101; zero them for the kinds above ---- */
    const int32_t *indices2;      /* CF/FC Jacobi: the F-points (indices = the C-points) */
    int64_t n_indices2;
    int32_t f_iterations;         /* CF/FC Jacobi: F sweeps per iteration */
    int32_t c_iterations;         /* CF/FC Jacobi: C sweeps per iteration */
    const double *coefficients;   /* polynomial: coefficients of p in DESCENDING order (relaxation.py:606-617) */
    int32_t n_coefficients;
    int32_t reserved_;
} amgb_smoother;

const char *amgb_last_error(void);
int amgb_version(void);
int amgb_device_count(void);

/* ---- (1) hierarchy + cycle driver ----------------------------------------------------------- */
int amgb_hierarchy_create(int device, amgb_hierarchy **out);
void amgb_hierarchy_destroy(amgb_hierarchy *h);

/* Append level k (call in order k = 0, 1, ...).  For every level but the last pass P, R and the
 * two smoothers; for the coarsest pass P = R = NULL (smoothers ignored). Arrays are copied to
 * HBM before the call returns. */
int amgb_hierarchy_add_level(amgb_hierarchy *h, const amgb_matrix *A, const amgb_matrix *P,
                             const amgb_matrix *R, const amgb_smoother *pre,
                             const amgb_smoother *post);

/* Coarsest-level solver: dense pseudo-inverse (n x n row-major) computed by the caller on the
 * CPU (scipy.linalg.pinv, multilevel.py:717-721) and applied on the GPU.  coarse_is_zero != 0
 * reproduces GenericSolver.__call__'s "A.nnz == 0 => x = 0" branch (multilevel.py:801-803). */
int amgb_hierarchy_set_coarse_pinv(amgb_hierarchy *h, int32_t n, const double *pinv,
                                   int32_t coarse_is_zero);

/* Coarsest-level solver = relaxation (multilevel.py:764-781: coarse_solver='gauss_seidel' | 'jacobi' | 'sor' |
 * 'block_jacobi' | 'block_gauss_seidel' | 'richardson' | 'chebyshev', default 10 iterations): x = 0, then the
 * smoother `sm` applied once (its `iterations` sweeps).  Call after the last amgb_hierarchy_add_level instead of
 * amgb_hierarchy_set_coarse_pinv. */
int amgb_hierarchy_set_coarse_relaxation(amgb_hierarchy *h, const amgb_smoother *sm);

/* Allocate work vectors, build wave schedules, capture CUDA graphs.  stream == NULL -> the
 * engine's own stream; otherwise every launch goes to the caller's stream (a cudaStream_t). */
int amgb_hierarchy_finalize(amgb_hierarchy *h, void *stream);

/* MultilevelSolver.solve without accel (multilevel.py:398-582): HOST b (n), HOST x (in: x0,
 * out: solution), stop when ||b - A x|| < tol * ||b|| (||b|| := 1 if 0) tested after each cycle, or
 * after maxiter cycles.  residuals (if non-NULL) receives ||r_0||, ||r_1||, ... (maxiter+1 slots);
 * *n_residuals its count; *info = 0 on convergence else the iteration count (:574-582). */
int amgb_solve(amgb_hierarchy *h, const double *b_host, double *x_host, double tol,
               int32_t maxiter, int32_t cycle, int32_t cycles_per_level, double *residuals,
               int32_t *n_residuals, int32_t *info);

/* amgb_solve with flags: AMGB_FLAG_X0_ZERO = the initial guess is zero, x_host is output only (saves the
 * host->device copy of x0; what aspreconditioner() and solve(x0=None) need). */
#define AMGB_FLAG_X0_ZERO 1
#define AMGB_FLAG_FLEXIBLE 2   /* amgb_solve_gmres: flexible GMRES (pyamg.krylov.fgmres) instead of pyamg.krylov.gmres */
#define AMGB_FLAG_MGS 8        /* amgb_solve_gmres: modified Gram-Schmidt GMRES (pyamg.krylov.gmres_mgs); not with FLEXIBLE */
#define AMGB_FLAG_REORTH 16    /* with AMGB_FLAG_MGS: gmres_mgs(reorth=True), a second MGS pass when ||v|| dropped */
/* AMGB_FLAG_DEVICE_IO, accepted by amgb_solve_ex, amgb_solve_cg, amgb_solve_bicgstab, amgb_solve_gmres,
 * amgb_solve_krylov and the five amgb_solve_many* entries: b / x (B / X, n x k row-major) are DEVICE pointers (device or managed memory on the
 * hierarchy's device), read and written in place without host staging; residuals, n_residuals and info stay host
 * arrays.  x / X is the initial guess unless AMGB_FLAG_X0_ZERO, and always the output.  Each pointer is checked
 * (cudaPointerGetAttributes) before anything is enqueued: anything else is AMGB_EINVAL.  The call orders itself
 * against the stream set by amgb_hierarchy_set_io_stream: its reads of b / x follow the work enqueued there before
 * the call, and work enqueued there after the call follows its writes of x.
 * amgb_solve_ex and amgb_solve_many with tol == 0 and residuals == NULL never wait for the device: they enqueue the
 * cycles and return, with *info = maxiter and *n_residuals = maxiter + 1 (the one-cycle preconditioner, maxiter = 1,
 * is such a call).  With tol > 0 they read one norm per cycle on the host, and the Krylov entries read their
 * per-iteration scalars on the host, as without the flag. */
#define AMGB_FLAG_DEVICE_IO 4
/* The caller's stream for AMGB_FLAG_DEVICE_IO calls (a cudaStream_t on the hierarchy's device; cudaStreamLegacy for
 * the legacy default stream).  NULL (the initial value) = the hierarchy's own stream, i.e. no cross-stream ordering.
 * Ordering uses one event each way, none when the two streams are the same; no other stream is synchronised. */
int amgb_hierarchy_set_io_stream(amgb_hierarchy *h, void *stream);
int amgb_solve_ex(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t maxiter,
                  int32_t cycle, int32_t cycles_per_level, int32_t flags, double *residuals,
                  int32_t *n_residuals, int32_t *info);

/* MultilevelSolver.solve(accel='cg') with every vector resident in HBM: pyamg's preconditioned CG
 * (pyamg/krylov/_cg.py:97-196, criteria 'rr') with M = one multigrid cycle from x0 = 0
 * (aspreconditioner, multilevel.py:355-396).  residuals: maxiter+1 slots; *info: 0 converged,
 * k = maxiter reached, -1 = indefinite matrix / preconditioner detected (the reference's warning). */
int amgb_solve_cg(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t maxiter,
                  int32_t cycle, int32_t flags, double *residuals, int32_t *n_residuals, int32_t *info);

/* MultilevelSolver.solve(accel='gmres' | 'fgmres') with every long vector resident in HBM: pyamg's Householder
 * GMRES (pyamg/krylov/_gmres_householder.py:21-360 -- what pyamg.krylov.gmres resolves to; left-preconditioned,
 * stops on the preconditioned residual against ||M b||) or, with AMGB_FLAG_FLEXIBLE, its flexible GMRES
 * (pyamg/krylov/_fgmres.py:17-345; right-preconditioned), M = one multigrid cycle from x0 = 0.
 * restart = 0: no restarts, at most `maxiter` inner iterations (maxiter <= 0: min(n, 40)); restart > 0: `maxiter`
 * outer iterations of `restart` inner ones (:129-149).  residuals: caller-sized (max_residuals slots),
 * *n_residuals = the number the method produced; *info: 0 converged, -1 stagnated (:339-346), else the number
 * of inner iterations performed.  Needs n >= 2 (n == 1 is a closed form, :152-154).
 * With AMGB_FLAG_MGS the method is pyamg's modified Gram-Schmidt GMRES (pyamg/krylov/_gmres_mgs.py:42-342; left-
 * preconditioned, stops on the preconditioned residual against ||M b||, same restart / maxiter meaning and residual
 * contract); AMGB_FLAG_REORTH adds its reorth=True pass.  MGS | FLEXIBLE, and REORTH without MGS, are AMGB_EINVAL. */
int amgb_solve_gmres(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t restart,
                     int32_t maxiter, int32_t cycle, int32_t flags, double *residuals, int32_t max_residuals,
                     int32_t *n_residuals, int32_t *info);

/* MultilevelSolver.solve(accel='bicgstab') resident in HBM: pyamg's right-preconditioned BiCGStab
 * (pyamg/krylov/_bicgstab.py:10-200, criteria 'rr') with M = one multigrid cycle from x0 = 0.  residuals:
 * maxiter+1 slots; *info: 0 converged, else maxiter.  Needs n >= 2. */
int amgb_solve_bicgstab(amgb_hierarchy *h, const double *b_host, double *x_host, double tol, int32_t maxiter,
                        int32_t cycle, int32_t flags, double *residuals, int32_t *n_residuals, int32_t *info);

/* MultilevelSolver.solve(accel='cgnr' | 'cgne' | 'minimal_residual' | 'steepest_descent') resident in HBM: pyamg's
 * CGNR (pyamg/krylov/_cgnr.py:97-220), CGNE (_cgne.py:97-214), minimal residual (_minimal_residual.py:92-163) or
 * steepest descent (_steepest_descent.py:92-197), criteria 'rr', with M = one multigrid cycle from x0 = 0.
 * method: one of the AMGB_KRYLOV_* constants.  residuals: maxiter+1 slots (minimal residual records ||M r||, the
 * others ||r||); *info: 0 converged, maxiter reached, or -1 with *reason saying why (AMGB_REASON_*).  flags:
 * AMGB_FLAG_X0_ZERO, AMGB_FLAG_DEVICE_IO.  CGNR and CGNE apply A^H: call amgb_hierarchy_set_transpose0 first
 * (AMGB_ESTATE otherwise). */
#define AMGB_KRYLOV_CGNR 0
#define AMGB_KRYLOV_CGNE 1
#define AMGB_KRYLOV_MR 2
#define AMGB_KRYLOV_SD 3
#define AMGB_REASON_NONE 0
#define AMGB_REASON_INDEFINITE_MATRIX 1
#define AMGB_REASON_INDEFINITE_PRECONDITIONER 2
#define AMGB_REASON_SINGULAR_PRECONDITIONER 3
int amgb_solve_krylov(amgb_hierarchy *h, int32_t method, const double *b_host, double *x_host, double tol,
                      int32_t maxiter, int32_t cycle, int32_t flags, double *residuals, int32_t *n_residuals,
                      int32_t *info, int32_t *reason);

/* A^H of the fine-level operator (CSR, or BSR expanded like level 0; row i = column i of A in ascending row order of
 * A), for CGNR and CGNE.  Copied to HBM in level-0 numbering before the call returns; replaces an earlier one and is
 * freed with the hierarchy.  Costs about the device memory of level 0's operator.  Call after finalize. */
int amgb_hierarchy_set_transpose0(amgb_hierarchy *h, const amgb_matrix *AH);

/* A new fine-level matrix under a finalized hierarchy (MultilevelSolver.change_solve_matrix, pyamg/multilevel.py:
 * 320-337): level 0 becomes A with the smoothers pre / post (A's shape; every other level, P_0 / R_0 on the level-1
 * side and the coarse solver stay).  Every later solve returns what a hierarchy finalized from scratch on the same
 * levels returns, bit for bit.  *path says what was done:
 *   1 = values refreshed in place: A has the pattern level 0 was built from, pre / post have the same kind, sweep,
 *       iterations, row lists, block size and polynomial degree as before (omega, Dinv and coefficients may differ),
 *       and the new values take the same value stream (fp64 / value / pair / row codes).  Level 0's permutation,
 *       waves, tiles, P_0 and R_0 stay; A's values (8 B per entry) and codes and the smoothers' Dinv go up, and the
 *       normal-equation / Schwarz sorted copies are refilled on the device.  The first such call downloads level 0's
 *       pattern to compare with and keeps the caller's (4 B per entry of host memory).
 *   2 = level 0 rebuilt: its layout, tiles and codes from A and the smoothers, P_0 / R_0 renumbered from their device
 *       copies.
 * The A^H of amgb_hierarchy_set_transpose0 is dropped (set it again before CGNR / CGNE) and captured cycles are
 * captured again on their next use.  Work goes to `stream` (NULL = the hierarchy's stream) after the hierarchy's
 * stream has drained; the call returns when it is complete.  AMGB_ENOTIMPL: a one-level hierarchy (level 0 is the
 * coarse level; nothing changed).  AMGB_EINVAL: A's shape differs.  Any other failure after the checks leaves the
 * hierarchy unusable (AMGB_ESTATE on every solve): destroy it. */
int amgb_hierarchy_replace_level0(amgb_hierarchy *h, const amgb_matrix *A, const amgb_smoother *pre,
                                  const amgb_smoother *post, void *stream, int32_t *path);

/* The same on DEVICE vectors (no host copies): x_dev in/out, b_dev in. Runs exactly `ncycles`
 * cycles (tol = 0 semantics); if norms2_dev != NULL it receives ncycles+1 squared residual norms. */
int amgb_solve_device(amgb_hierarchy *h, const double *b_dev, double *x_dev, int32_t ncycles,
                      int32_t cycle, int32_t cycles_per_level, double *norms2_dev);

/* amgb_solve_ex on k right-hand sides at once: B_host / X_host are n x k row-major (NumPy C order of an (n, k)
 * array), column j is solved as amgb_solve_ex would solve it (its own ||b||, stop test and info; a column that
 * converges keeps the iterate of that cycle).  Up to eight columns share each pass over the hierarchy.
 * residuals: (maxiter+1) x k row-major, n_residuals and info: k entries (each may be NULL).
 * AMGB_ENOTIMPL (nothing computed): a smoother, or a relaxation coarse solver, other than none / Jacobi /
 * Gauss-Seidel / block Jacobi / block Gauss-Seidel / polynomial, or an AMLI cycle -- solve such hierarchies column
 * by column. */
int amgb_solve_many(amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host, double tol,
                    int32_t maxiter, int32_t cycle, int32_t cycles_per_level, int32_t flags, double *residuals,
                    int32_t *n_residuals, int32_t *info);

/* amgb_solve_cg / amgb_solve_bicgstab on k right-hand sides at once (MultilevelSolver.solve_many(accel='cg' |
 * 'bicgstab')): column j -- iterate, residual list and info -- is what the single-vector entry computes on column j,
 * with up to eight columns per pass over the hierarchy.  Layout as amgb_solve_many: B_host / X_host n x k row-major
 * (X_host is the initial guess unless AMGB_FLAG_X0_ZERO), residuals (maxiter+1) x k row-major, n_residuals and info
 * k entries (each may be NULL).  AMGB_ENOTIMPL (nothing computed) in the cases amgb_solve_many rejects.
 * amgb_solve_many_bicgstab needs n >= 2. */
int amgb_solve_many_cg(amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host, double tol,
                       int32_t maxiter, int32_t cycle, int32_t flags, double *residuals, int32_t *n_residuals,
                       int32_t *info);
int amgb_solve_many_bicgstab(amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host, double tol,
                             int32_t maxiter, int32_t cycle, int32_t flags, double *residuals, int32_t *n_residuals,
                             int32_t *info);

/* amgb_solve_gmres on k right-hand sides at once (MultilevelSolver.solve_many(accel='gmres' | 'fgmres')): column j
 * -- iterate, residual list and info -- is what amgb_solve_gmres computes on column j with the same tol, restart,
 * maxiter, cycle and flags (AMGB_FLAG_X0_ZERO | AMGB_FLAG_FLEXIBLE | AMGB_FLAG_MGS | AMGB_FLAG_REORTH, validated as
 * there), with up to eight columns per pass over the
 * hierarchy.  B_host / X_host n x k row-major, residuals max_residuals x k row-major, n_residuals and info k entries
 * (each may be NULL).  AMGB_ENOTIMPL (nothing computed) in the cases amgb_solve_many rejects, and when not even two
 * columns' reflector store fits in device memory; the hierarchy stays usable.  Needs n >= 2. */
int amgb_solve_many_gmres(amgb_hierarchy *h, int32_t k, const double *B_host, double *X_host, double tol,
                          int32_t restart, int32_t maxiter, int32_t cycle, int32_t flags, double *residuals,
                          int32_t max_residuals, int32_t *n_residuals, int32_t *info);

/* amgb_solve_krylov on k right-hand sides at once (MultilevelSolver.solve_many(accel='cgnr' | 'cgne' |
 * 'minimal_residual' | 'steepest_descent')): column j -- iterate, residual list, info and reason -- is what
 * amgb_solve_krylov computes on column j, with up to eight columns per pass over the hierarchy.  Layout as
 * amgb_solve_many_cg: B_host / X_host n x k row-major, residuals (maxiter+1) x k row-major, n_residuals, info and
 * reason k entries (each may be NULL).  AMGB_ENOTIMPL (nothing computed) in the cases amgb_solve_many rejects. */
int amgb_solve_many_krylov(amgb_hierarchy *h, int32_t method, int32_t k, const double *B_host, double *X_host,
                           double tol, int32_t maxiter, int32_t cycle, int32_t flags, double *residuals,
                           int32_t *n_residuals, int32_t *info, int32_t *reason);

/* amgb_solve_device on k columns: B_dev / X_dev are n x k row-major device arrays (X_dev in/out); if
 * norms2_dev != NULL it receives (ncycles+1) x k squared residual norms.  Same scope as amgb_solve_many. */
int amgb_solve_many_device(amgb_hierarchy *h, int32_t k, const double *B_dev, double *X_dev, int32_t ncycles,
                           int32_t cycle, int32_t cycles_per_level, double *norms2_dev);

/* One multigrid cycle x <- cycle(x, b) on the engine's level-0 device vectors / introspection */
int amgb_hierarchy_num_levels(const amgb_hierarchy *h);
int64_t amgb_hierarchy_device_bytes(const amgb_hierarchy *h);
/* kernels launched by the most recent amgb_solve / amgb_solve_device call */
int64_t amgb_hierarchy_last_launches(const amgb_hierarchy *h);
/* One un-graphed cycle with a CUDA-event pair around every operator launch (measurement aid).
 * rec[6k..6k+5] = level, op (0 spmv, 1 residual, 2 prolong+add, 3 jacobi, 4 gs wave, 5 block jacobi,
 * 6 coarse tail = all levels below in one cluster kernel, rows = #steps),
 * rows, nnz, algorithmic bytes (SURVEY.md 8(d) formulas), milliseconds. */
int amgb_profile_cycle(amgb_hierarchy *h, int32_t cycle, double *rec, int32_t max_records,
                       int32_t *n_records);
/* pinned host buffers for the e2e path (cudaHostAlloc / cudaFreeHost) */
int amgb_host_alloc(size_t bytes, void **out);
int amgb_host_free(void *p);

/* ---- (1b) one resident operator (tile kernels) on device vectors ----------------------------- */
typedef struct amgb_operator amgb_operator;
/* Upload M (CSR/BSR host arrays) and build its TMA tiles.  wave_ptr (n_waves+1 entries, or NULL) marks
 * contiguous row ranges that are mutually independent Gauss-Seidel waves (tiles never cross them). */
int amgb_operator_create(int device, const amgb_matrix *M, const int64_t *wave_ptr, int32_t n_waves,
                         void *stream, amgb_operator **out);
void amgb_operator_destroy(amgb_operator *op);
/* kind: 0 y = M x | 1 y = b - M x (+ |y|^2 -> norm2_out) | 2 y += M x | 3 y = jacobi(x; b, omega), r = b - M x
 * (r optional) | 4 Gauss-Seidel sweep of wave `wave`, in place on y (pass x == y).  DEVICE pointers; x must
 * hold M.n_cols entries followed by at least 2 readable doubles (16-byte TMA reads). */
int amgb_operator_apply(amgb_operator *op, int32_t kind, const double *x, const double *b, double *y,
                        double *r, double omega, double *norm2_out, int32_t wave);

/* ---- (2) reference-FFI-shaped host entry points --------------------------------------------- */
/* amg_core.jacobi (relaxation.h:309-346) */
int amgb_host_jacobi(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                     const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                     int b_size, double *temp, int temp_size, int32_t row_start,
                     int32_t row_stop, int32_t row_step, const double *omega, int omega_size);
/* amg_core.gauss_seidel (relaxation.h:48-76) -- executed as dependency waves, same result */
int amgb_host_gauss_seidel(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                           const double *Ax, int Ax_size, double *x, int x_size,
                           const double *b, int b_size, int32_t row_start, int32_t row_stop,
                           int32_t row_step);
/* amg_core.sor_gauss_seidel (relaxation.h:116-145) */
int amgb_host_sor_gauss_seidel(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                               const double *Ax, int Ax_size, double *x, int x_size,
                               const double *b, int b_size, int32_t row_start, int32_t row_stop,
                               int32_t row_step, double omega);
/* amg_core.gauss_seidel_indexed (relaxation.h:736-768) */
int amgb_host_gauss_seidel_indexed(const int32_t *Ap, int Ap_size, const int32_t *Aj,
                                   int Aj_size, const double *Ax, int Ax_size, double *x,
                                   int x_size, const double *b, int b_size, const int32_t *Id,
                                   int Id_size, int32_t row_start, int32_t row_stop,
                                   int32_t row_step);
/* amg_core.bsr_jacobi (relaxation.h:472-562) */
int amgb_host_bsr_jacobi(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                         const double *Ax, int Ax_size, double *x, int x_size, const double *b,
                         int b_size, double *temp, int temp_size, int32_t row_start,
                         int32_t row_stop, int32_t row_step, int32_t blocksize,
                         const double *omega, int omega_size);
/* amg_core.block_jacobi (relaxation.h:1021-1090) */
int amgb_host_block_jacobi(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                           const double *Ax, int Ax_size, double *x, int x_size,
                           const double *b, int b_size, const double *Tx, int Tx_size,
                           double *temp, int temp_size, int32_t row_start, int32_t row_stop,
                           int32_t row_step, const double *omega, int omega_size,
                           int32_t blocksize);
/* amg_core.jacobi_indexed (relaxation_bind.cpp:164-196 <- relaxation.h:382-427) */
int amgb_host_jacobi_indexed(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                             const double *Ax, int Ax_size, double *x, int x_size,
                             const double *b, int b_size, const int32_t *indices, int indices_size,
                             const double *omega, int omega_size);
/* amg_core.block_gauss_seidel (relaxation_bind.cpp:545-580 <- relaxation.h:1242-1298); only the full forward
 * (0, nb, 1) and backward (nb-1, -1, -1) ranges the reference's Python layer passes (relaxation.py:561-582) */
int amgb_host_block_gauss_seidel(const int32_t *Ap, int Ap_size, const int32_t *Aj, int Aj_size,
                                 const double *Ax, int Ax_size, double *x, int x_size,
                                 const double *b, int b_size, const double *Tx, int Tx_size,
                                 int32_t row_start, int32_t row_stop, int32_t row_step, int32_t blocksize);
/* One application of ANY smoother descriptor to host vectors (x in place): what calling a level's
 * presmoother(A, x, b) does in the reference (multilevel.py:610).  Runs the same wave schedules, tiles and
 * kernels the cycle uses; the entry point behind the Python mirrors of relaxation.polynomial / cf_jacobi /
 * fc_jacobi / jacobi_indexed / block_gauss_seidel. */
int amgb_host_relax(const amgb_matrix *A, const amgb_smoother *sm, double *x, const double *b);
/* GPU-resident Arnoldi rounds for the spectral-radius estimates of the smoother setup (pyamg/util/linalg.py:255-383
 * approximate_spectral_radius -> _approximate_eigenvalues :90-252): the operator x -> diag(row_scale) (A x)
 * (row_scale may be NULL) is uploaded once; amgb_arnoldi_run does a whole round of modified-Gram-Schmidt Arnoldi
 * on the device and returns the (maxiter+1) x maxiter Hessenberg matrix (row-major) and the number of valid steps;
 * the host picks the restart vector from H's eigen-decomposition and hands its coefficients in the (still resident)
 * basis to amgb_arnoldi_combine; the next run with v0_host == NULL starts from it. */
typedef struct amgb_arnoldi amgb_arnoldi;
int amgb_arnoldi_create(int device, const amgb_matrix *A, const double *row_scale, int32_t maxiter, amgb_arnoldi **out);
int amgb_arnoldi_run(amgb_arnoldi *a, const double *v0_host, double breakdown, double *H_host, int32_t *m_done);
int amgb_arnoldi_combine(amgb_arnoldi *a, const double *coef, int32_t m);
void amgb_arnoldi_destroy(amgb_arnoldi *a);

/* scipy.sparse._sparsetools.csr_matmat as the setup phase uses it for the Galerkin product `R @ A @ P`
 * (pyamg/classical/classical.py:201, pyamg/aggregation/aggregation.py:425): C = A B with SciPy's results bit for
 * bit -- same summation order per entry, same (reverse first-appearance) column order inside a row, exact zeros
 * dropped.  CSR operands (block 1x1).  The three output arrays are malloc'ed by the library: release them with
 * amgb_free.  Rows with more than 8192 products: AMGB_ENOTIMPL. */
int amgb_host_csr_matmat(const amgb_matrix *A, const amgb_matrix *B, int32_t **Cp, int32_t **Cj, double **Cx,
                         int64_t *nnz);
void amgb_free(void *p);
/* pyamg.graph.vertex_coloring(G, 'MIS') (pyamg/graph.py:84-126 -> amg_core vertex_coloring_mis, graph.h:218-235)
 * computed on the device: same colours vertex by vertex (structurally symmetric pattern; the diagonal is ignored).
 * rounds (nullable): wavefront rounds used. */
int amgb_host_vertex_coloring_mis(int32_t n, const int32_t *Ap, const int32_t *Aj, int32_t *colors,
                                  int32_t *n_colors, int32_t *rounds);
/* scipy.sparse._sparsetools.csr_matvec / bsr_matvec as the cycle uses them (y = A x) */
int amgb_host_matvec(const amgb_matrix *A, const double *x, double *y);

/* ---- (3) device kernels ------------------------------------------------------------------- */
/* lanes: lanes per row (power of two 1..32), 0 = choose from the mean row length */
int amgb_dev_csr_spmv(int32_t n_rows, const int32_t *Ap, const int32_t *Aj, const double *Ax,
                      const double *x, double *y, int lanes, void *stream);
/* r = b - A x; partials (>= amgb_dev_partials_len(n_rows, lanes) doubles) may be NULL */
int amgb_dev_csr_residual(int32_t n_rows, const int32_t *Ap, const int32_t *Aj,
                          const double *Ax, const double *x, const double *b, double *r,
                          double *partials, double *norm2_out, int lanes, void *stream);
/* x += P xc */
int amgb_dev_csr_spmv_add(int32_t n_rows, const int32_t *Ap, const int32_t *Aj,
                          const double *Ax, const double *xc, double *x, int lanes, void *stream);
/* fused Jacobi + residual: x_out = jacobi(x_in), r_out (nullable) = b - A x_in */
int amgb_dev_csr_jacobi(int32_t n_rows, const int32_t *Ap, const int32_t *Aj, const double *Ax,
                        const double *x_in, const double *b, double *x_out, double *r_out,
                        double omega, int lanes, void *stream);
/* Gauss-Seidel over an independent set: rows == NULL -> rows row0 .. row0+n-1 */
int amgb_dev_csr_gs_wave(int32_t n, int32_t row0, const int32_t *rows, const int32_t *Ap,
                         const int32_t *Aj, const double *Ax, double *x, const double *b,
                         double omega, int lanes, void *stream);
int64_t amgb_dev_partials_len(int32_t n_rows, int lanes);
int amgb_dev_dense_matvec(int32_t m, int32_t n, const double *M, const double *x, double *y,
                          void *stream);
int amgb_dev_fill(double *x, int64_t n, double v, void *stream);
/* out_dev[0] = <x, y> (x == y: squared 2-norm) by the engine's deterministic two-stage reduction (the `norm2` of
 * SURVEY.md 8(b)); scratch = amgb_dev_reduce_len() doubles of device memory. */
int64_t amgb_dev_reduce_len(void);
int amgb_dev_dot(const double *x, const double *y, int64_t n, double *scratch, double *out_dev, void *stream);
/* y = a x + b y */
int amgb_dev_axpby(double a, const double *x, double b, double *y, int64_t n, void *stream);
/* bsr_block_jacobi of SURVEY.md 8(b) on the point-CSR expansion of the BSR operator (Ap has n_block_rows*bs + 1
 * entries), Dinv (n_block_rows, bs, bs) row-major, bs <= 8, x_out != x_in. */
int amgb_dev_block_jacobi(int32_t n_block_rows, int32_t bs, const int32_t *Ap, const int32_t *Aj, const double *Ax,
                          const double *x_in, const double *b, const double *Dinv, double *x_out, double omega,
                          int lanes, void *stream);
/* out[i] = in[idx[i]] (halo packing, permuted layouts) */
int amgb_dev_gather(const double *in, const int32_t *idx, double *out, int64_t n, void *stream);
/* HOST helper (no CUDA): the TMA tile list for a CSR row-pointer array under geometry (T, RMAX), G lanes per
 * row and optional row breaks; row0/nz0 get n_tiles+1 descriptors (sentinel last). For tests of the tiling rules. */
int amgb_debug_build_tiles(int32_t n, const int32_t *Ap, int32_t G, const int64_t *breaks, int32_t n_breaks,
                           int32_t T, int32_t RMAX, int32_t *row0, int32_t *nz0, int32_t cap, int32_t *tile_ptr,
                           int32_t *n_tiles);
/* HOST helper (no CUDA): dependency waves of the sequential sweep over `list` (NULL = 0..n-1);
 * wave_of[k] is the 1-based wave of list position k. */
int amgb_wave_schedule(int32_t n, const int32_t *Ap, const int32_t *Aj, const int32_t *list, int64_t m,
                       int32_t *wave_of, int32_t *n_waves);

/* ---- (4) multi-GPU halo exchange over NVLink peer memory (SURVEY.md 8(e): the reference has no distributed
 *      path; this replaces the host-issued ncclAllGather per operator application of round 1) -----------------
 * One process per GPU.  amgb_comm_create allocates this rank's IPC block (flags + double-buffered staging for
 * `cap_doubles` halo entries) and returns 64 opaque handle bytes; the ranks exchange the handles (any transport:
 * torch.distributed all_gather) and amgb_comm_connect maps the blocks of the ranks in nbr_mask (bit q = rank q
 * is a halo neighbour at some level; the masks must be symmetric).  amgb_comm_exchange is ONE kernel on the
 * communicator's stream: packed boundary entries of v are stored straight into the neighbours' staging buffers,
 * a flag per source rank is released system-wide, the kernel waits for its own sources and unpacks into the halo
 * region of v ([owned (n_own) | from rank 0 | from rank 1 | ...]).  Graph-capturable (no host work, no NCCL). */
typedef struct amgb_comm amgb_comm;
int amgb_comm_create(int device, int world, int rank, int64_t cap_doubles, void *stream, amgb_comm **out,
                     unsigned char *handle64);
int amgb_comm_connect(amgb_comm *c, const unsigned char *handles /* world x 64 bytes */, uint32_t nbr_mask);
/* send_idx: DEVICE array of local indices packed per destination rank; send_off: HOST, world + 1 offsets into it;
 * peer_off: HOST, world entries: where this rank's block starts in destination q's halo region; recv_total:
 * entries this rank receives. */
int amgb_comm_exchange(amgb_comm *c, double *v, int64_t n_own, const int32_t *send_idx, const int64_t *send_off,
                       const int64_t *peer_off, int64_t recv_total);
void amgb_comm_destroy(amgb_comm *c);

#ifdef __cplusplus
}
#endif
#endif /* PYAMG_B200_H */
