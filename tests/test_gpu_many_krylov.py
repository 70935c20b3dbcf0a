"""MultilevelSolver.solve_many(accel='cg' | 'bicgstab'): the GPU-resident Krylov methods on k right-hand sides per
pass over the hierarchy (amgb_solve_many_cg / amgb_solve_many_bicgstab).

Column j of a batched Krylov solve must be exactly what solve(B[:, j], accel=...) returns -- iterate, info and
residual list, bit for bit: the batched cycle, SpMVs, dot products and vector updates keep the single path's
per-row and per-reduction order.  Column 0 is also checked against the reference goldens like solve itself.
"""
import os
import warnings

import numpy as np
import pytest

from conftest import GOLDEN, GOLDEN_DIR, relerr, summation_order_sensitivity

pytestmark = pytest.mark.gpu
METHODS = ("cg", "bicgstab")
BICGSTAB = dict(tol=1e-10, maxiter=8)        # test_oracle.KRYLOV_RUNS["bicgstab"]
BICGSTAB_W = dict(tol=1e-4, maxiter=20, cycle="W")


def _block(ex, n, seed=5):
    b = ex["b"].ravel()
    return np.column_stack([b, np.random.default_rng(seed).standard_normal(n), np.zeros(n), -2.0 * b])


def _per_column(ml, B, X0=None, **kw):
    xs, infos, lists = [], [], []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for j in range(B.shape[1]):
            rj = []
            xj, ij = ml.solve(B[:, j], x0=None if X0 is None else X0[:, j].copy(), residuals=rj, return_info=True,
                              **kw)
            xs.append(xj)
            infos.append(ij)
            lists.append(rj)
    return np.column_stack(xs), infos, lists


def _many_equals_per_column(ml, B, X0=None, rel=None, **kw):
    """solve_many(accel=...) against per-column solve: bit for bit, or (rel set) to that relative difference with
    the same info and residual-list lengths."""
    res = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X, info = ml.solve_many(B, X0=X0, residuals=res, return_info=True, **kw)
    assert X.shape == B.shape and X.dtype == np.float64 and X.flags.c_contiguous
    Xr, ir, rr = _per_column(ml, B, X0, **kw)
    assert len(res) == B.shape[1]
    for j in range(B.shape[1]):
        assert info[j] == ir[j], j
        if rel is None:
            assert np.array_equal(X[:, j], Xr[:, j]), j
            assert res[j] == rr[j], j
        else:
            assert relerr(X[:, j], Xr[:, j]) < rel and len(res[j]) == len(rr[j]), j
    return X, info, res


@pytest.mark.parametrize("name", GOLDEN)
def test_columns_match_golden_and_solve_cg(name, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n)
    X, info, res = _many_equals_per_column(ml, B, tol=1e-10, maxiter=10, accel="cg")
    if "x_ref_cg" in ex:
        assert relerr(X[:, 0], ex["x_ref_cg"]) < 1e-11
        assert info[0] == int(ex["info_cg"][0]) and len(res[0]) == len(ex["residuals_cg"])
    assert info[2] == 0 and len(res[2]) == 1 and not X[:, 2].any()      # zero column: stops at once


@pytest.mark.parametrize("name", GOLDEN)
def test_columns_match_golden_and_solve_bicgstab(name, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    kg = np.load(os.path.join(GOLDEN_DIR, "krylov", name + ".npz"))
    B = _block(ex, n)
    X, info, res = _many_equals_per_column(ml, B, accel="bicgstab", **BICGSTAB)
    assert info[0] == int(kg["info_bicgstab"][0]) and len(res[0]) == len(kg["residuals_bicgstab"])
    bound = max(1e-9, 20 * summation_order_sensitivity(ml, ex["b"], accel="bicgstab", **BICGSTAB))
    assert relerr(X[:, 0], kg["x_ref_bicgstab"]) < bound
    assert info[2] == 0 and len(res[2]) == 1 and not X[:, 2].any()


@pytest.mark.parametrize("name", GOLDEN)
def test_w_cycle_with_x0(name, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n)[:, :3]                  # k = 3: one group padded to K = 4
    X0 = np.column_stack([ex["x0"].ravel(), np.random.default_rng(7).standard_normal(n), np.zeros(n)])
    X0_copy = X0.copy()
    X, info, res = _many_equals_per_column(ml, B, X0=X0, tol=1e-3, maxiter=30, cycle="W", accel="cg")
    assert np.array_equal(X0, X0_copy)
    if "x_ref_cgW" in ex:
        assert relerr(X[:, 0], ex["x_ref_cgW"]) < 1e-11
        assert info[0] == int(ex["info_cgW"][0]) and len(res[0]) == len(ex["residuals_cgW"])
    kg = np.load(os.path.join(GOLDEN_DIR, "krylov", name + ".npz"))
    X, info, res = _many_equals_per_column(ml, B, X0=X0, accel="bicgstab", **BICGSTAB_W)
    assert np.array_equal(X0, X0_copy)
    assert info[0] == int(kg["info_bicgstabW"][0]) and len(res[0]) == len(kg["residuals_bicgstabW"])
    bound = max(1e-9, 20 * summation_order_sensitivity(ml, ex["b"], x0=ex["x0"], accel="bicgstab", **BICGSTAB_W))
    assert relerr(X[:, 0], kg["x_ref_bicgstabW"]) < bound


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg2_sa_jacobi_poisson2d", "cfg5_sa_bjacobi_elasticity"])
def test_columns_stop_at_different_iterations(name, method, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(11)
    b = ex["b"].ravel()
    B = np.column_stack([b, rng.standard_normal(n), np.zeros(n), b + 1e-3 * rng.standard_normal(n), 1e-8 * b])
    X0 = np.column_stack([ex["x0"].ravel(), np.zeros(n), np.zeros(n), rng.standard_normal(n), np.zeros(n)])
    X, info, res = _many_equals_per_column(ml, B, X0=X0, tol=1e-6, maxiter=40, accel=method)
    assert info[2] == 0 and len(res[2]) == 1 and not X[:, 2].any()
    assert len({len(r) for r in res}) > 1


def test_indefinite_operator_returns_minus_one_and_warns_once():
    from pyamg_b200.aggregation import smoothed_aggregation_solver
    from pyamg_b200.gallery import poisson
    A = -poisson((40, 40), format="csr")
    ml = smoothed_aggregation_solver(A, max_coarse=20)
    n = A.shape[0]
    B = np.column_stack([np.random.default_rng(s).standard_normal(n) for s in range(3)] + [np.zeros(n)])
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        X, info = ml.solve_many(B, tol=1e-8, maxiter=20, accel="cg", return_info=True)
    indefinite = [w for w in caught if "Indefinite" in str(w.message)]
    assert len(indefinite) == 1
    assert list(info[:3]) == [-1, -1, -1] and info[3] == 0
    _many_equals_per_column(ml, B, tol=1e-8, maxiter=20, accel="cg")


def test_nonsymmetric_smoothing_warns_once(load_golden):
    for name in GOLDEN:
        ml, ex = load_golden(name)
        if not ml.symmetric_smoothing:
            break
    else:
        pytest.skip("every cfg1-6 hierarchy smooths symmetrically")
    B = _block(ex, ml.levels[0].A.shape[0])
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        ml.solve_many(B, tol=1e-10, maxiter=3, accel="cg")
    assert len([w for w in caught if "non-symmetric" in str(w.message)]) == 1


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg5_sa_bjacobi_elasticity"])
@pytest.mark.parametrize("k", [1, 2, 3, 5, 8, 11])
def test_widths_and_groups(name, k, method, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(k).standard_normal((n, k))
    X, info, res = _many_equals_per_column(ml, B, tol=1e-10, maxiter=5, accel=method)
    assert X.shape == (n, k) and len(info) == k


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
    B = _block(ex, n)[:, :3]
    # a larger coarse tail makes solve's preconditioner run the tail as one cluster kernel, while the batched cycle
    # always issues the per-launch chain (DESIGN 5e): the two agree to rounding there, not bit for bit
    rel = 1e-9 if "AMGB_TAIL_NNZ" in env else None
    X, info, res = _many_equals_per_column(ml, B, rel=rel, tol=1e-10, maxiter=10, accel="cg")
    if "x_ref_cg" in ex:
        assert relerr(X[:, 0], ex["x_ref_cg"]) < 1e-11
    _many_equals_per_column(ml, B, rel=rel, accel="bicgstab", **BICGSTAB)


@pytest.mark.parametrize("name,kw", [("cfg9_air_fcjacobi_advection2d", dict(accel="cg")),
                                     ("cfg9_air_fcjacobi_advection2d", dict(accel="bicgstab")),
                                     ("cfg3_rs_mcgs_poisson3d", dict(accel="fgmres", cycle="AMLI")),
                                     ("cfg2_sa_jacobi_poisson2d", dict(accel="gmres"))])
def test_fallback_equals_per_column_solve(name, kw, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(4).standard_normal((n, 3))
    _many_equals_per_column(ml, B, tol=1e-8, maxiter=6, **kw)
    single = ml.last_launches()        # the last engine call solved one column
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ml.solve(B[:, 2], tol=1e-8, maxiter=6, **kw)
    assert ml.last_launches() == single


def test_batched_launches_versus_single_cg(load_golden):
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(3).standard_normal((n, 4))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ml.solve(B[:, 0], tol=0, maxiter=3, accel="cg")
        single = ml.last_launches()
        ml.solve_many(B, tol=0, maxiter=3, accel="cg")
    assert ml.last_launches() < 2 * single


def test_validation_and_defaults(load_golden):
    ml, ex = load_golden("cfg2_sa_jacobi_poisson2d")
    n = ml.levels[0].A.shape[0]
    B = np.column_stack([ex["b"].ravel(), np.ones(n)])
    for method in METHODS:
        with pytest.raises(ValueError):
            ml.solve_many(B, maxiter=0, accel=method)
        with pytest.raises(ValueError):
            ml.solve_many(B, X0=np.ones((n, 3)), accel=method)
        with pytest.raises(NotImplementedError):
            ml.solve_many(B.astype(complex), accel=method)
        # maxiter=None: the per-method default of solve
        _many_equals_per_column(ml, B, tol=1e-8, maxiter=None, accel=method)
    with pytest.raises(ValueError):            # AMLI needs fgmres, as in solve
        ml.solve_many(B, accel="cg", cycle="AMLI")
