"""MultilevelSolver.solve_many on the hierarchies users build by default: block Gauss-Seidel (the smoothed-aggregation
and root-node default, scalar and elasticity), polynomial smoothers (Chebyshev / Richardson) and relaxation coarse
solvers, batched K-wide like Jacobi / Gauss-Seidel / block Jacobi (tests/test_gpu_many.py).

Column j of a batched solve must be exactly what solve() returns on column j -- iterate, info and residual list, bit
for bit -- for plain cycling and for accel='cg' | 'bicgstab'.  Column 0 is also checked against the reference's stored
results and every column against the oracle.
"""
import os
import warnings

import numpy as np
import pytest

import oracle
import pyamg_b200
from conftest import GOLDEN_DIR, golden_path, relerr

pytestmark = pytest.mark.gpu
TOL = 1e-12

CFG7 = "cfg7_sa_cheby_richardson_poisson2d"
CFG10 = "cfg10_sa_bgs_elasticity"
CFG11 = "cfg11_rs_gs_coarse_relaxation"
CFGS = [CFG7, CFG10, CFG11]
ADOPTED = ["sa_default", "rootnode", "sa_elasticity_default", "sa_energy_chebyshev", "rs_coarse_gauss_seidel"]
SPD = [CFG7, CFG10, "sa_default", "sa_elasticity_default"]
WIDTHS = [3, 5, 8, 11]          # padding to 4 and 8, a full group, more than one group


def _load(name):
    from pyamg_b200.hierarchy_io import load_hierarchy
    if name in ADOPTED:
        stored, ex = load_hierarchy(os.path.join(GOLDEN_DIR, "adopt", name + ".npz"))
        return pyamg_b200.MultilevelSolver.from_pyamg(stored), ex
    return load_hierarchy(golden_path(name))


@pytest.fixture(scope="module")
def hier():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _load(name)
        return cache[name]

    return get


def _device_bytes(ml):
    from pyamg_b200 import _engine as E
    return int(E.lib().amgb_hierarchy_device_bytes(ml.handle))


def _block(ex, n, k=4, seed=5):
    """Column 0 the stored right-hand side, column 2 zero, the others random or a multiple of column 0."""
    rng = np.random.default_rng(seed)
    b = np.asarray(ex["b"], dtype=float).ravel()
    cols = [b, rng.standard_normal(n), np.zeros(n), -2.0 * b] + [rng.standard_normal(n) for _ in range(max(k - 4, 0))]
    return np.column_stack(cols[:k])


def _equals_per_column(ml, B, X0=None, **kw):
    """solve_many against solve on every column: iterate, info and residual list bit for bit."""
    res = []
    before = _device_bytes(ml)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X, info = ml.solve_many(B, X0=X0, residuals=res, return_info=True, **kw)
        batched_bytes = _device_bytes(ml)
        assert X.shape == B.shape and X.dtype == np.float64 and X.flags.c_contiguous
        assert len(res) == B.shape[1]
        for j in range(B.shape[1]):
            rj = []
            xj, ij = ml.solve(B[:, j], x0=None if X0 is None else X0[:, j].copy(), residuals=rj, return_info=True, **kw)
            assert np.array_equal(X[:, j], xj), j
            assert info[j] == ij, j
            assert list(res[j]) == list(rj), j
    return X, info, res, batched_bytes - before


@pytest.mark.parametrize("name", CFGS + ADOPTED)
def test_columns_match_reference_oracle_and_solve(name, hier):
    ml, ex = hier(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n)
    its = 3 if name in ADOPTED else len(ex["residuals"]) - 1
    fresh = ml._h is None
    X, info, res, grew = _equals_per_column(ml, B, tol=0, maxiter=its)
    if fresh:
        assert grew > 0            # the K-wide level blocks were allocated: the hierarchy ran batched, not by fallback
    assert relerr(X[:, 0], ex["x_V3" if name in ADOPTED else "x_ref"]) < TOL
    assert list(info) == [its] * 4 and all(len(r) == its + 1 for r in res)
    assert not X[:, 2].any()       # a zero column stays exactly zero
    cyc = oracle.Cycle(oracle.hierarchy_spec(ml), coarse_pinv=ml.coarse_solver.P)
    for j in range(B.shape[1]):
        assert relerr(X[:, j], cyc.solve(B[:, j], tol=0, maxiter=its)) < TOL


@pytest.mark.parametrize("name", CFGS + ADOPTED)
def test_w_and_f_cycles(name, hier):
    ml, ex = hier(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n, k=3)          # one group padded to K = 4
    X = _equals_per_column(ml, B, tol=0, maxiter=2, cycle="W")[0]
    assert relerr(X[:, 0], ex["x_W2" if name in ADOPTED else "x_ref_W"]) < TOL
    X = _equals_per_column(ml, B, tol=0, maxiter=2, cycle="F")[0]
    if name not in ADOPTED:
        assert relerr(X[:, 0], ex["x_ref_F"]) < TOL
    _equals_per_column(ml, B, tol=0, maxiter=2, cycle="F", cycles_per_level=2)


@pytest.mark.parametrize("k", WIDTHS)
@pytest.mark.parametrize("name", CFGS)
def test_widths_and_groups(name, k, hier):
    ml, ex = hier(name)
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(k).standard_normal((n, k))
    X, info, res, _ = _equals_per_column(ml, B, tol=0, maxiter=3)
    assert X.shape == (n, k) and list(info) == [3] * k


@pytest.mark.parametrize("name", CFGS + ["sa_default", "rs_coarse_gauss_seidel"])
def test_tolerance_stop_per_column_with_x0(name, hier):
    ml, ex = hier(name)
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(11)
    b = np.asarray(ex["b"], dtype=float).ravel()
    x0 = np.asarray(ex["x0"], dtype=float).ravel() if "x0" in ex else rng.standard_normal(n)
    B = np.column_stack([b, rng.standard_normal(n), np.zeros(n), b + 1e-3 * rng.standard_normal(n), 1e-6 * b])
    X0 = np.column_stack([x0, np.zeros(n), np.zeros(n), rng.standard_normal(n), 1e-6 * x0])
    X0_copy = X0.copy()
    X, info, res, _ = _equals_per_column(ml, B, X0=X0, tol=1e-6, maxiter=50)
    assert np.array_equal(X0, X0_copy)
    if "x_ref_tol" in ex:
        assert info[0] == int(ex["info_tol"][0]) and len(res[0]) == len(ex["residuals_tol"])
        assert relerr(X[:, 0], ex["x_ref_tol"]) < TOL
    assert info[2] == 0 and len(res[2]) == 2 and not X[:, 2].any()      # a zero column stops after one cycle
    assert len({len(r) for r in res}) > 1                                # columns stop at different cycles


@pytest.mark.parametrize("method", ["cg", "bicgstab"])
@pytest.mark.parametrize("name", SPD)
def test_krylov_columns_equal_solve(name, method, hier):
    ml, ex = hier(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n, k=5)
    X, info, res, _ = _equals_per_column(ml, B, tol=1e-10, maxiter=10, accel=method)
    if method == "cg" and "x_ref_cg" in ex:
        assert relerr(X[:, 0], ex["x_ref_cg"]) < 1e-11
        assert info[0] == int(ex["info_cg"][0]) and len(res[0]) == len(ex["residuals_cg"])
    assert info[2] == 0 and len(res[2]) == 1 and not X[:, 2].any()      # zero column: stops at once
    rng = np.random.default_rng(12)
    X0 = np.column_stack([rng.standard_normal(n), np.zeros(n), np.zeros(n)])
    _equals_per_column(ml, B[:, :3], X0=X0, tol=1e-4, maxiter=20, cycle="W", accel=method)


@pytest.mark.parametrize("name", [CFG10, CFG7])
def test_batched_launches_versus_fallback(name, hier):
    ml, ex = hier(name)
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(3).standard_normal((n, 4))
    ml.solve(B[:, 0], tol=0, maxiter=3)
    single = ml.last_launches()
    ml.solve_many(B, tol=0, maxiter=3)
    assert ml.last_launches() < 2 * single


@pytest.mark.parametrize("env", [{"AMGB_NO_GRAPH": "1"}, {"AMGB_NO_PERMUTE": "1"}, {"AMGB_NO_TILES": "1"},
                                 {"AMGB_TILE_MIN_NNZ": "0"}])
@pytest.mark.parametrize("name", [CFG10, CFG7])
def test_kernel_paths(name, env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ml, ex = _load(name)            # the switches are read when the hierarchy is uploaded
    n = ml.levels[0].A.shape[0]
    its = len(ex["residuals"]) - 1
    X = _equals_per_column(ml, _block(ex, n, k=3), tol=0, maxiter=its)[0]
    assert relerr(X[:, 0], ex["x_ref"]) < TOL
    X = _equals_per_column(ml, _block(ex, n, k=3), tol=0, maxiter=2, cycle="W")[0]
    assert relerr(X[:, 0], ex["x_ref_W"]) < TOL


def _polynomial_levels(ml):
    """Indices of the levels that smooth (or coarse-solve) with a polynomial."""
    spec = oracle.hierarchy_spec(ml)
    out = []
    for l, d in enumerate(spec):
        kinds = [s[0] for s in (d.get("pre"), d.get("post"), d.get("coarse_relax")) if s is not None]
        if "polynomial" in kinds:
            out.append(l)
    return out


@pytest.mark.parametrize("name", [CFG7, "sa_energy_chebyshev", CFG10])
def test_device_bytes_grow_by_the_horner_blocks_only_with_polynomial_smoothers(name):
    """The K-wide buffers of a hierarchy against those of the same hierarchy with Jacobi smoothers: two more n x K
    blocks on every level that smooths with a polynomial, nothing more anywhere else."""
    from pyamg_b200.relaxation.smoothing import change_smoothers
    ml, ex = _load(name)
    plain, _ = _load(name)
    change_smoothers(plain, "jacobi", "jacobi")
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(2).standard_normal((n, 4))
    grew = []
    for m in (ml, plain):
        before = _device_bytes(m)
        m.solve_many(B, tol=0, maxiter=1)
        grew.append(_device_bytes(m) - before)
    poly = _polynomial_levels(ml)
    assert bool(poly) == (name != CFG10)
    block = lambda rows: (8 * (rows * 4 + 2) + 255) // 256 * 256      # noqa: E731  (one K = 4 level block)
    assert grew[1] > 0
    assert grew[0] - grew[1] == sum(2 * block(ml.levels[l].A.shape[0]) for l in poly)
