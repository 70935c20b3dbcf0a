"""MultilevelSolver.solve_many: k right-hand sides per pass over the hierarchy (amgb_solve_many).

Column j of a batched solve must be what solve() computes on column j: the batched kernels keep the per-row
summation order of the single-vector kernels, so the two agree to rounding (and are checked against the
reference goldens and the oracle like solve itself).
"""
import numpy as np
import pytest

import oracle
from conftest import GOLDEN, relerr

pytestmark = pytest.mark.gpu
TOL = 1e-12


def _block(ex, n, seed=5):
    b = ex["b"].ravel()
    return np.column_stack([b, np.random.default_rng(seed).standard_normal(n), np.zeros(n), -2.0 * b])


def _col_close(a, b, rel=1e-14):
    nb = np.linalg.norm(b)
    return np.linalg.norm(a - b) <= rel * (nb if nb > 0 else 1.0)


@pytest.mark.parametrize("name", GOLDEN)
def test_columns_match_reference_oracle_and_solve(name, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    its = len(ex["residuals"]) - 1
    B = _block(ex, n)
    res = []
    X = ml.solve_many(B, tol=0, maxiter=its, residuals=res)
    assert X.shape == B.shape and X.dtype == np.float64 and X.flags.c_contiguous
    assert relerr(X[:, 0], ex["x_ref"]) < TOL
    cyc = oracle.Cycle(oracle.hierarchy_spec(ml), coarse_pinv=ml.coarse_solver.P)
    assert len(res) == B.shape[1]
    for j in range(B.shape[1]):
        rj = []
        xj = ml.solve(B[:, j], tol=0, maxiter=its, residuals=rj)
        assert relerr(X[:, j], cyc.solve(B[:, j], tol=0, maxiter=its)) < TOL
        assert _col_close(X[:, j], xj)
        assert len(res[j]) == len(rj) == its + 1
        assert np.allclose(res[j], rj, rtol=1e-12, atol=1e-13 * max(rj[0], 1e-300))
    assert not X[:, 2].any()


@pytest.mark.parametrize("name", GOLDEN)
def test_w_and_f_cycles_with_padding(name, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n)[:, :3]          # k = 3: one group padded to K = 4
    for cyc, ref in (("W", "x_ref_W"), ("F", "x_ref_F")):
        X = ml.solve_many(B, tol=0, maxiter=2, cycle=cyc)
        assert relerr(X[:, 0], ex[ref]) < TOL
        assert _col_close(X[:, 1], ml.solve(B[:, 1], tol=0, maxiter=2, cycle=cyc))


@pytest.mark.parametrize("name", GOLDEN)
def test_tolerance_stop_per_column_with_x0(name, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(11)
    b = ex["b"].ravel()
    B = np.column_stack([b, rng.standard_normal(n), np.zeros(n), b + 1e-3 * rng.standard_normal(n)])
    X0 = np.column_stack([ex["x0"].ravel(), np.zeros(n), np.zeros(n), rng.standard_normal(n)])
    X0_copy = X0.copy()
    res = []
    X, info = ml.solve_many(B, X0=X0, tol=1e-6, maxiter=50, residuals=res, return_info=True)
    assert np.array_equal(X0, X0_copy)
    assert info[0] == int(ex["info_tol"][0])
    assert len(res[0]) == len(ex["residuals_tol"])
    assert relerr(X[:, 0], ex["x_ref_tol"]) < TOL
    assert info[2] == 0 and len(res[2]) == 2 and not X[:, 2].any()      # a zero column stops after one cycle
    for j in (1, 3):
        rj = []
        xj, ij = ml.solve(B[:, j], x0=X0[:, j].copy(), tol=1e-6, maxiter=50, residuals=rj, return_info=True)
        assert info[j] == ij and len(res[j]) == len(rj)
        assert _col_close(X[:, j], xj)


@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg5_sa_bjacobi_elasticity"])
@pytest.mark.parametrize("k", [1, 2, 3, 5, 8, 11])
def test_widths_and_groups(name, k, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(k).standard_normal((n, k))
    X, info = ml.solve_many(B, tol=0, maxiter=3, return_info=True)
    assert X.shape == (n, k) and list(info) == [3] * k
    for j in range(k):
        assert _col_close(X[:, j], ml.solve(B[:, j], tol=0, maxiter=3))


@pytest.mark.parametrize("env", [{"AMGB_NO_TILES": "1"}, {"AMGB_NO_PERMUTE": "1"}, {"AMGB_NO_GRAPH": "1"},
                                 {"AMGB_TILE_MIN_NNZ": "0", "AMGB_TILE_FLAT": "0"},
                                 {"AMGB_TILE_MIN_NNZ": "0", "AMGB_TILE_FLAT": "2"},
                                 {"AMGB_TILE_MIN_NNZ": "0", "AMGB_TILE_DENSE_CFG": "7", "AMGB_TILE_DENSE_AVG": "4"},
                                 {"AMGB_TAIL_NNZ": "600000"}])
@pytest.mark.parametrize("name", ["cfg3_rs_mcgs_poisson3d", "cfg5_sa_bjacobi_elasticity"])
def test_kernel_paths(name, env, monkeypatch):
    from pyamg_b200.hierarchy_io import load_hierarchy
    from conftest import golden_path
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ml, ex = load_hierarchy(golden_path(name))
    n = ml.levels[0].A.shape[0]
    its = len(ex["residuals"]) - 1
    B = _block(ex, n)[:, :3]
    X = ml.solve_many(B, tol=0, maxiter=its)
    assert relerr(X[:, 0], ex["x_ref"]) < TOL
    for j in range(3):
        assert _col_close(X[:, j], ml.solve(B[:, j], tol=0, maxiter=its))
    assert relerr(ml.solve_many(B, tol=0, maxiter=2, cycle="W")[:, 0], ex["x_ref_W"]) < TOL


def test_batched_launches_versus_fallback(load_golden):
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(3).standard_normal((n, 4))
    ml.solve(B[:, 0], tol=0, maxiter=3)
    single = ml.last_launches()
    ml.solve_many(B, tol=0, maxiter=3)
    assert ml.last_launches() < 2 * single


@pytest.mark.parametrize("name,cycle", [("cfg9_air_fcjacobi_advection2d", "V"), ("cfg3_rs_mcgs_poisson3d", "AMLI")])
def test_fallback_equals_per_column_solve(name, cycle, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(4).standard_normal((n, 3))
    res = []
    X, info = ml.solve_many(B, tol=1e-8, maxiter=4, cycle=cycle, residuals=res, return_info=True)
    last = ml.last_launches()          # the last engine call solved one column
    for j in range(3):
        rj = []
        xj, ij = ml.solve(B[:, j], tol=1e-8, maxiter=4, cycle=cycle, residuals=rj, return_info=True)
        assert np.array_equal(X[:, j], xj) and info[j] == ij and res[j] == rj
    assert ml.last_launches() == last


def test_validation(load_golden):
    ml, ex = load_golden("cfg2_sa_jacobi_poisson2d")
    n = ml.levels[0].A.shape[0]
    B = np.ones((n, 2))
    with pytest.raises(ValueError):
        ml.solve_many(np.ones(n))
    with pytest.raises(ValueError):
        ml.solve_many(np.ones((n + 1, 2)))
    with pytest.raises(ValueError):
        ml.solve_many(B, X0=np.ones((n, 3)))
    with pytest.raises(ValueError):
        ml.solve_many(B, maxiter=0)
    with pytest.raises(NotImplementedError):
        ml.solve_many(B.astype(complex))


def test_device_entry_matches_host_entry(load_golden):
    import ctypes
    import torch
    from pyamg_b200 import _engine as E
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(8).standard_normal((n, 5))
    X0 = np.random.default_rng(9).standard_normal((n, 5))
    res = []
    Xh = ml.solve_many(B, X0=X0, tol=0, maxiter=3, residuals=res)
    dev = "cpu" if E.lib().amgb_device_count() < 1 or not torch.cuda.is_available() else "cuda"
    Bd = torch.from_numpy(B).to(dev)
    Xd = torch.from_numpy(X0).to(dev)
    N2 = torch.zeros((4, 5), dtype=torch.float64, device=dev)
    if dev == "cuda":
        torch.cuda.synchronize()        # the engine runs on its own stream
    E.check(E.lib().amgb_solve_many_device(ml.handle, 5, Bd.data_ptr(), Xd.data_ptr(), 3, 0, 1, N2.data_ptr()))
    if dev == "cuda":
        torch.cuda.synchronize()
    assert np.array_equal(Xd.cpu().numpy(), Xh)
    assert np.allclose(np.sqrt(N2.cpu().numpy()), np.array(res).T, rtol=1e-12)
