"""MultilevelSolver.solve_many on hierarchies smoothed by the normal-equation smoothers (jacobi_ne, gauss_seidel_ne,
gauss_seidel_nr) and by overlapping Schwarz (schwarz, strength_based_schwarz), batched K-wide like the other smoothers
(tests/test_gpu_many.py, tests/test_gpu_many_widening.py).

Column j of a batched solve must be exactly what solve() returns on column j -- iterate, info and residual list, bit
for bit -- for plain cycling, for the batched accelerators and for CUDA tensors.  Column 0 is also checked against the
reference's stored results and every column against the oracle.  Every test also shows that the batched path ran: the
hierarchy's device bytes grow by the K-wide level blocks, which a column-by-column fallback never allocates.
"""
import warnings

import numpy as np
import pytest

import oracle
from conftest import golden_path, relerr

pytestmark = pytest.mark.gpu
TOL = 1e-12

CFG13 = "cfg13_rs_gsnr_gsne_advdiff2d"          # gauss_seidel_nr symmetric / gauss_seidel_ne backward
CFG14 = "cfg14_sa_jacobine_poisson2d"           # jacobi_ne
CFG15 = "cfg15_sa_schwarz_aniso2d"              # schwarz
CFG16 = "cfg16_sa_strength_schwarz_aniso2d"     # strength_based_schwarz
CFGS = [CFG13, CFG14, CFG15, CFG16]
WIDTHS = [3, 5, 8, 11]          # padding to 4 and 8, a full group, more than one group


def _load(name):
    from pyamg_b200.hierarchy_io import load_hierarchy
    return load_hierarchy(golden_path(name))


def _device_bytes(ml):
    from pyamg_b200 import _engine as E
    return int(E.lib().amgb_hierarchy_device_bytes(ml.handle))


def _level_blocks(ml, K):
    """Bytes of the four K-wide vector blocks (x, x', b, r) of every level: what a batched solve of width K adds."""
    return sum(4 * ((8 * (lvl.A.shape[0] * K + 2) + 255) // 256 * 256) for lvl in ml.levels)


def _block(ex, n, k=4, seed=5):
    """Column 0 the stored right-hand side, column 2 zero, the others random or a multiple of column 0."""
    rng = np.random.default_rng(seed)
    b = np.asarray(ex["b"], dtype=float).ravel()
    cols = [b, rng.standard_normal(n), np.zeros(n), -2.0 * b] + [rng.standard_normal(n) for _ in range(max(k - 4, 0))]
    return np.column_stack(cols[:k])


def _solve_many(ml, B, X0=None, **kw):
    res = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X, info = ml.solve_many(B, X0=X0, residuals=res, return_info=True, **kw)
    return X, info, res


def _equals_per_column(ml, B, X0=None, norms_rtol=None, **kw):
    """solve_many against solve on every column: iterate, info and residual list bit for bit (the residual list to
    norms_rtol when that is given).  solve runs once first, so that whatever it allocates is in place; returns X,
    info, residual lists and how many device bytes the batched call added."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ml.solve(B[:, 0], x0=None if X0 is None else X0[:, 0].copy(), **kw)
    before = _device_bytes(ml)
    X, info, res = _solve_many(ml, B, X0, **kw)
    grew = _device_bytes(ml) - before
    assert X.shape == B.shape and X.dtype == np.float64
    assert len(res) == B.shape[1]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for j in range(B.shape[1]):
            rj = []
            xj, ij = ml.solve(B[:, j], x0=None if X0 is None else X0[:, j].copy(), residuals=rj, return_info=True,
                              **kw)
            assert np.array_equal(X[:, j], xj), j
            assert info[j] == ij, j
            if norms_rtol is None:
                assert list(res[j]) == list(rj), j
            else:
                assert np.allclose(res[j], rj, rtol=norms_rtol, atol=0), j
    return X, info, res, grew


def _ran_batched(ml, k, grew):
    K = 2 if k <= 2 else (4 if k <= 4 else 8)
    assert grew >= _level_blocks(ml, K), (grew, _level_blocks(ml, K))


def _oracle(ml):
    return oracle.Cycle(oracle.hierarchy_spec(ml), coarse_pinv=getattr(ml.coarse_solver, "P", None))


@pytest.mark.parametrize("k", WIDTHS)
@pytest.mark.parametrize("name", CFGS)
def test_columns_match_reference_oracle_and_solve(name, k):
    ml, ex = _load(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n, k=k, seed=k)
    its = len(ex["residuals"]) - 1
    X, info, res, grew = _equals_per_column(ml, B, tol=0, maxiter=its)
    _ran_batched(ml, k, grew)
    assert relerr(X[:, 0], ex["x_ref"]) < TOL
    assert list(info) == [its] * k and all(len(r) == its + 1 for r in res)
    assert not X[:, 2].any()       # a zero column stays exactly zero
    cyc = _oracle(ml)
    for j in range(k):
        assert relerr(X[:, j], cyc.solve(B[:, j], tol=0, maxiter=its)) < TOL
    for cycle, ref in (("W", "x_ref_W"), ("F", "x_ref_F")):
        X = _equals_per_column(ml, B, tol=0, maxiter=2, cycle=cycle)[0]
        assert relerr(X[:, 0], ex[ref]) < TOL, cycle
        for j in range(k):
            assert relerr(X[:, j], cyc.solve(B[:, j], tol=0, maxiter=2, cycle=cycle)) < TOL, (cycle, j)
    _equals_per_column(ml, B[:, :3], tol=0, maxiter=2, cycle="F", cycles_per_level=2)


@pytest.mark.parametrize("name", CFGS)
def test_tolerance_stop_per_column_with_x0(name):
    ml, ex = _load(name)
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(11)
    b = np.asarray(ex["b"], dtype=float).ravel()
    x0 = np.asarray(ex["x0"], dtype=float).ravel()
    B = np.column_stack([b, rng.standard_normal(n), np.zeros(n), b + 1e-3 * rng.standard_normal(n), 1e-6 * b])
    X0 = np.column_stack([x0, np.zeros(n), np.zeros(n), rng.standard_normal(n), 1e-6 * x0])
    X, info, res, grew = _equals_per_column(ml, B, X0=X0, tol=1e-6, maxiter=50)
    _ran_batched(ml, 5, grew)
    assert info[2] == 0 and len(res[2]) == 2 and not X[:, 2].any()      # a zero column stops after one cycle


ACCELS = [(CFG13, m) for m in ("gmres", "fgmres", "bicgstab", "cgnr")] + \
         [(c, m) for c in (CFG14, CFG15, CFG16) for m in ("cg", "gmres", "minimal_residual")]


@pytest.mark.parametrize("name,method", ACCELS)
def test_accelerated_columns_equal_solve(name, method):
    ml, ex = _load(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n, k=5)
    X, info, res, grew = _equals_per_column(ml, B, tol=1e-10, maxiter=8, accel=method)
    _ran_batched(ml, 5, grew)
    assert info[2] == 0 and len(res[2]) == 1 and not X[:, 2].any()      # zero column: stops at once
    rng = np.random.default_rng(12)
    X0 = np.column_stack([rng.standard_normal(n), np.zeros(n), np.zeros(n)])
    _equals_per_column(ml, B[:, :3], X0=X0, tol=1e-4, maxiter=10, cycle="W", accel=method)


# ------------------------------------------------------------------ this repository's host setup, every sweep
def _host_sa(grid, pre, post, coarse="pinv", seed=21):
    from pyamg_b200.aggregation import smoothed_aggregation_solver
    from pyamg_b200.gallery import poisson
    from pyamg_b200.relaxation.smoothing import change_smoothers
    np.random.seed(seed)
    ml = smoothed_aggregation_solver(poisson((grid, grid), format="csr"), max_coarse=40, coarse_solver=coarse)
    change_smoothers(ml, pre, post)
    return ml


SWEEPS = [(("gauss_seidel_nr", {"sweep": s, "iterations": it}), ("gauss_seidel_ne", {"sweep": t, "iterations": 3 - it}))
          for s, t, it in (("forward", "backward", 1), ("backward", "symmetric", 2), ("symmetric", "forward", 1),
                           ("symmetric", "symmetric", 2))] + \
         [(("jacobi_ne", {"iterations": it, "omega": 0.8}), ("gauss_seidel_nr", {"sweep": "forward"})) for it in (1, 2)] + \
         [(("schwarz", {"sweep": s, "iterations": it}), ("strength_based_schwarz", {"sweep": t, "iterations": 3 - it}))
          for s, t, it in (("forward", "backward", 1), ("backward", "symmetric", 2), ("symmetric", "forward", 2))]
COARSE = [("gauss_seidel_nr", {"sweep": "symmetric", "iterations": 3}),
          ("gauss_seidel_ne", {"sweep": "backward", "iterations": 2}),
          ("jacobi_ne", {"iterations": 4}),
          ("schwarz", {"sweep": "symmetric", "iterations": 2})]


def _host_case(ml, k):
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(k).standard_normal((n, k))
    B[:, 1] = 0.0
    X, info, res, grew = _equals_per_column(ml, B, tol=0, maxiter=3)
    _ran_batched(ml, k, grew)
    assert not X[:, 1].any()
    cyc = _oracle(ml)
    for j in range(k):
        assert relerr(X[:, j], cyc.solve(B[:, j], tol=0, maxiter=3)) < TOL, j
    _equals_per_column(ml, B, tol=0, maxiter=2, cycle="W")


@pytest.mark.parametrize("case", range(len(SWEEPS)))
def test_host_setup_every_sweep(case):
    pre, post = SWEEPS[case]
    _host_case(_host_sa(20, pre, post), 5)


@pytest.mark.parametrize("coarse", COARSE, ids=[c[0] for c in COARSE])
def test_relaxation_coarse_solvers(coarse):
    ml = _host_sa(20, ("gauss_seidel_nr", {"sweep": "symmetric"}), ("schwarz", {"sweep": "backward"}), coarse=coarse)
    assert ml.coarse_solver.relaxation is not None and ml.levels[-1].A.shape[0] > 1
    _host_case(ml, 3)


# ------------------------------------------------------------------ forced kernel paths
# 560 x 560: the level-0 operators (A and the smoothers' copies of it, 1.57 M entries) are above the default tile
# threshold and the coarser ones below it, so the default mixes tile and rows launches; AMGB_TILE_MIN_NNZ=0 sends
# every operator through the tile kernel, AMGB_NO_TILES every one through the rows kernel, AMGB_NO_GRAPH issues the
# batched cycle launch by launch instead of replaying its graph
@pytest.fixture(scope="module")
def large():
    cache = {}

    def get(smoothers):
        if smoothers not in cache:
            if smoothers == "ne":
                pre, post = ("gauss_seidel_nr", {"sweep": "symmetric"}), ("jacobi_ne", {"iterations": 2})
            else:
                pre, post = ("schwarz", {"sweep": "symmetric"}), ("gauss_seidel_ne", {"sweep": "backward"})
            cache[smoothers] = _host_sa(560, pre, post)
        return cache[smoothers]

    return get


@pytest.mark.parametrize("env", [{}, {"AMGB_TILE_MIN_NNZ": "0"}, {"AMGB_NO_TILES": "1"}, {"AMGB_NO_GRAPH": "1"}],
                         ids=["default", "tiles", "no_tiles", "no_graph"])
@pytest.mark.parametrize("smoothers", ["ne", "schwarz"])
def test_kernel_paths(smoothers, env, large, monkeypatch):
    for key, v in env.items():
        monkeypatch.setenv(key, v)
    ml = large(smoothers)
    ml._invalidate()                        # the switches are read when the hierarchy is uploaded
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(7).standard_normal((n, 3))
    # iterates bit for bit; the level-0 residual norms to rounding: where that operator has tiles, the batched
    # residual-norm launch groups its K-wide partial sums by its own grid, not by the single tile kernel's
    X, info, res, grew = _equals_per_column(ml, B, norms_rtol=1e-14, tol=0, maxiter=2)
    _ran_batched(ml, 3, grew)
    _equals_per_column(ml, B, norms_rtol=1e-14, tol=0, maxiter=1, cycle="W")
    ml._invalidate()


# ------------------------------------------------------------------ CUDA tensors
def _torch_cuda():
    try:
        import torch
    except ImportError:
        return None
    return torch if torch.cuda.is_available() else None


@pytest.mark.skipif(_torch_cuda() is None, reason="needs torch with a CUDA device")
@pytest.mark.parametrize("name", [CFG13, CFG15])
def test_cuda_tensor_blocks_equal_host_blocks(name):
    torch = _torch_cuda()
    ml, ex = _load(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n, k=5)
    X0 = np.random.default_rng(3).standard_normal((n, 5))
    before = _device_bytes(ml)                       # a tensor call first: it allocates the K = 8 blocks
    Xt, it, rt = _solve_many(ml, torch.from_numpy(B).cuda(), tol=1e-8, maxiter=5)
    torch.cuda.synchronize()
    assert _device_bytes(ml) - before >= _level_blocks(ml, 8)
    for kw in (dict(tol=1e-8, maxiter=5), dict(tol=0, maxiter=3, cycle="W"), dict(tol=1e-8, maxiter=6, accel="gmres"),
               dict(tol=1e-8, maxiter=6, accel="minimal_residual")):
        for x0 in (None, X0):
            Xh, ih, rh = _solve_many(ml, B, x0, **kw)
            Bt = torch.from_numpy(B).cuda()
            Xt, it, rt = _solve_many(ml, Bt, None if x0 is None else torch.from_numpy(x0).cuda(), **kw)
            torch.cuda.synchronize()
            assert isinstance(Xt, torch.Tensor) and Xt.is_cuda
            assert np.array_equal(Xt.cpu().numpy(), Xh), kw
            assert list(it) == list(ih) and [list(r) for r in rt] == [list(r) for r in rh], kw


# ------------------------------------------------------------------ Schwarz subdomains over the K-wide bound
def test_oversized_schwarz_subdomains_run_column_by_column():
    """A level-0 subdomain of 500 rows: 4 warps x 2 x 500 doubles = 32 KB per CTA for one column, 128 KB at K = 4 (above
    48 KB: the kernel's opt-in), 256 KB at K = 8, more than the 200 KB bound -- so a call whose widest group is 8
    columns wide solves column by column, and one of at most 4 columns runs batched."""
    n0 = 24 * 24
    sub = np.concatenate([np.arange(0, 500), np.arange(300, n0)]).astype(np.int32)
    ptr = np.array([0, 500, 500 + n0 - 300], dtype=np.int32)
    pre = [("schwarz", {"subdomain": sub, "subdomain_ptr": ptr, "sweep": "symmetric"}), ("gauss_seidel", {})]
    ml = _host_sa(24, pre, ("gauss_seidel_nr", {"sweep": "forward"}))
    assert ml.levels[0].A.shape[0] == n0
    rng = np.random.default_rng(9)
    for k, batched in ((3, True), (5, False), (11, False), (2, True)):
        B = rng.standard_normal((n0, k))
        X, info, res, grew = _equals_per_column(ml, B, tol=1e-8, maxiter=4)
        if batched:
            assert grew > 0, k
        else:
            assert grew == 0, k        # no K = 8 blocks: nothing ran batched
        cyc = _oracle(ml)
        assert relerr(X[:, 0], cyc.solve(B[:, 0], tol=1e-8, maxiter=4)) < TOL
    X, info, res, grew = _equals_per_column(ml, rng.standard_normal((n0, 6)), tol=1e-8, maxiter=4, accel="gmres")
    assert X.shape == (n0, 6)
