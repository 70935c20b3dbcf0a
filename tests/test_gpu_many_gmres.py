"""MultilevelSolver.solve_many(accel='gmres' | 'fgmres'): Householder GMRES and flexible GMRES on k right-hand sides
per pass over the hierarchy (amgb_solve_many_gmres).

Column j of a batched solve must be exactly what solve(B[:, j], accel=...) returns -- iterate, info and residual
list, bit for bit: the batched cycle, SpMVs, reductions and reflector kernels keep the single path's per-row and
per-reduction order.  Column 0 is also checked against the reference goldens like solve itself.
"""
import ctypes
import os
import warnings

import numpy as np
import pytest

from conftest import GOLDEN_ALL, GOLDEN_DIR, _cfg_number, golden_path, relerr, summation_order_sensitivity

pytestmark = pytest.mark.gpu
METHODS = ("gmres", "fgmres")
# the golden hierarchies amgb_solve_many batches, and those it leaves to solve
BATCHED = [g for g in GOLDEN_ALL if _cfg_number(g) <= 7 or _cfg_number(g) in (10, 11, 12)]
FALLBACK = [g for g in GOLDEN_ALL if _cfg_number(g) in (8, 9, 13, 14, 15, 16)]
GMRES_RUNS = ("gmres", "gmresW", "fgmres", "fgmresF")      # test_oracle.KRYLOV_RUNS entries without AMLI


def _device_bytes(ml):
    from pyamg_b200 import _engine as E
    return int(E.lib().amgb_hierarchy_device_bytes(ml.handle))


def _store_bytes(n, max_inner, flexible, K):
    npad = ((n + 2 + 31) // 32) * 32
    return (max_inner + 1 + (max_inner if flexible else 0)) * npad * K * 8


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


def _many_equals_per_column(ml, B, X0=None, **kw):
    """solve_many(accel=...) against per-column solve, bit for bit.  Returns X, info, residual lists and the
    hierarchy's device bytes right after the batched call."""
    res = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X, info = ml.solve_many(B, X0=X0, residuals=res, return_info=True, **kw)
    nbytes = _device_bytes(ml)
    assert X.shape == B.shape and X.dtype == np.float64 and X.flags.c_contiguous
    Xr, ir, rr = _per_column(ml, B, X0, **kw)
    assert len(res) == B.shape[1]
    for j in range(B.shape[1]):
        assert info[j] == ir[j], j
        assert np.array_equal(X[:, j], Xr[:, j]), j
        assert res[j] == rr[j], j
    return X, info, res, nbytes


def _block(ex, n, seed=5):
    b = ex["b"].ravel()
    return np.column_stack([b, np.random.default_rng(seed).standard_normal(n), np.zeros(n), -2.0 * b])


@pytest.mark.parametrize("name", BATCHED)
def test_columns_match_golden_and_solve(name):
    from pyamg_b200.hierarchy_io import load_hierarchy
    from test_oracle import KRYLOV_RUNS
    ml, ex = load_hierarchy(golden_path(name))            # fresh: the first batched call allocates the store
    n = ml.levels[0].A.shape[0]
    kg = np.load(os.path.join(GOLDEN_DIR, "krylov", name + ".npz"))
    B = _block(ex, n)
    x0 = ex["x0"].ravel()
    X0 = np.column_stack([x0, np.random.default_rng(6).standard_normal(n), np.zeros(n), -x0])
    before = _device_bytes(ml)
    for i, tag in enumerate(GMRES_RUNS):
        kw = dict(KRYLOV_RUNS[tag])
        with_x0 = tag in ("gmresW", "fgmresF")
        X, info, res, nbytes = _many_equals_per_column(ml, B, X0=X0 if with_x0 else None, **kw)
        if i == 0:                                         # the batched path ran: its reflector store is counted
            assert nbytes - before >= _store_bytes(n, min(kw["maxiter"], n), False, 4), tag
        assert info[0] == int(kg["info_" + tag][0]), tag
        assert len(res[0]) == len(kg["residuals_" + tag]), tag
        skw = dict(kw, x0=x0) if with_x0 else kw
        bound = max(1e-9, 20 * summation_order_sensitivity(ml, ex["b"], **skw))
        assert relerr(X[:, 0], kg["x_ref_" + tag]) < bound, tag
        if not with_x0:                                    # zero column, zero guess: stops at once
            assert info[2] == 0 and len(res[2]) == 1 and not X[:, 2].any(), tag


@pytest.mark.parametrize("name", FALLBACK)
def test_fallback_hierarchies_equal_per_column_solve(name, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n)[:, :3]
    for method in METHODS:
        _many_equals_per_column(ml, B, tol=1e-8, maxiter=6, accel=method)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg2_sa_jacobi_poisson2d", "cfg5_sa_bjacobi_elasticity"])
def test_columns_stop_at_different_inner_iterations(name, method, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(11)
    b = ex["b"].ravel()
    B = np.column_stack([b, rng.standard_normal(n), np.zeros(n), b + 1e-3 * rng.standard_normal(n), 1e-8 * b])
    X0 = np.column_stack([ex["x0"].ravel(), np.zeros(n), np.zeros(n), rng.standard_normal(n), np.zeros(n)])
    X, info, res, _ = _many_equals_per_column(ml, B, X0=X0, tol=1e-6, maxiter=40, accel=method)
    assert info[2] == 0 and len(res[2]) == 1 and not X[:, 2].any()
    assert len({len(r) for r in res}) > 1


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg5_sa_bjacobi_elasticity"])
@pytest.mark.parametrize("k", [2, 3, 5, 8, 11])
def test_widths_and_groups(name, k, method, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(k).standard_normal((n, k))
    X, info, res, _ = _many_equals_per_column(ml, B, tol=1e-10, maxiter=6, accel=method)
    assert X.shape == (n, k) and len(info) == k


def _c_gmres(ml, B, restart, maxiter, flags, tol=1e-12, rows=64):
    """amgb_solve_many_gmres on the block and amgb_solve_gmres per column, with the same C arguments."""
    from pyamg_b200 import _engine as E
    L = E.lib()
    n, k = B.shape
    Bh = np.ascontiguousarray(B)
    X = np.zeros((n, k))
    res = np.zeros((rows, k))
    nres, info = np.zeros(k, dtype=np.int32), np.zeros(k, dtype=np.int32)
    E.check(L.amgb_solve_many_gmres(ml.handle, k, Bh.ctypes.data, X.ctypes.data, tol, restart, maxiter,
                                    E.CYCLES["V"], flags, E.f64p(res), rows, E.i32p(nres), E.i32p(info)))
    for j in range(k):
        b = np.ascontiguousarray(B[:, j])
        x = np.zeros(n)
        r = np.zeros(rows)
        nr, inf = ctypes.c_int32(0), ctypes.c_int32(0)
        E.check(L.amgb_solve_gmres(ml.handle, b.ctypes.data, x.ctypes.data, tol, restart, maxiter, E.CYCLES["V"],
                                   flags, E.f64p(r), rows, ctypes.byref(nr), ctypes.byref(inf)))
        assert info[j] == inf.value and nres[j] == nr.value, j
        assert np.array_equal(X[:, j], x), j
        m = min(nr.value, rows)
        assert np.array_equal(res[:m, j], r[:m]), j
    return info, nres


@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg6_rs_gsfwd_none_poisson3d"])
def test_restarts_through_the_c_abi(name, load_golden):
    from pyamg_b200 import _engine as E
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n)
    for flags in (E.FLAG_X0_ZERO, E.FLAG_X0_ZERO | E.FLAG_FLEXIBLE):
        info, nres = _c_gmres(ml, B, restart=3, maxiter=4, flags=flags)
        assert nres[0] > 4                                 # more than one outer iteration ran


@pytest.mark.parametrize("env", [{"AMGB_NO_PERMUTE": "1"}, {"AMGB_NO_GRAPH": "1"}, {"AMGB_NO_TILES": "1"},
                                 {"AMGB_TILE_MIN_NNZ": "0"}])
@pytest.mark.parametrize("name", ["cfg3_rs_mcgs_poisson3d", "cfg5_sa_bjacobi_elasticity"])
def test_kernel_paths(name, env, monkeypatch):
    from pyamg_b200.hierarchy_io import load_hierarchy
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ml, ex = load_hierarchy(golden_path(name))
    n = ml.levels[0].A.shape[0]
    B = _block(ex, n)[:, :3]
    for method in METHODS:
        _many_equals_per_column(ml, B, tol=1e-10, maxiter=12, accel=method)


def test_reflector_store_narrows_to_what_fits():
    """Poisson 100^3 with maxiter=1500: eight columns would need about 96 GB of reflectors, more than the card
    holds, so the call runs at a narrower width -- with every column still equal to its single solve."""
    from pyamg_b200.classical import ruge_stuben_solver
    from pyamg_b200.gallery import poisson
    A = poisson((100, 100, 100), format="csr")
    ml = ruge_stuben_solver(A, max_coarse=500)
    n = A.shape[0]
    B = np.random.default_rng(8).standard_normal((n, 8))
    before = _device_bytes(ml)
    X, info, res, nbytes = _many_equals_per_column(ml, B, tol=1e-8, maxiter=1500, accel="gmres")
    assert (info == 0).all()
    assert nbytes - before < _store_bytes(n, 1500, False, 8)          # the 8-wide store was never kept
    assert nbytes - before >= _store_bytes(n, 1500, False, 2)
    # the hierarchy stays usable for both entry points
    x, i1 = ml.solve(B[:, 0], tol=1e-8, maxiter=50, return_info=True)
    assert i1 == 0
    X2, info2 = ml.solve_many(B[:, :3], tol=1e-8, maxiter=50, return_info=True)
    assert (info2 == 0).all() and np.array_equal(X2[:, 0], x)


def test_batched_launches_versus_single(load_golden):
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(3).standard_normal((n, 4))
    for method in METHODS:
        ml.solve(B[:, 0], tol=0, maxiter=6, accel=method)
        single = ml.last_launches()
        ml.solve_many(B, tol=0, maxiter=6, accel=method)
        assert ml.last_launches() < 4 * single, method


def test_validation_and_defaults(load_golden):
    ml, ex = load_golden("cfg2_sa_jacobi_poisson2d")
    n = ml.levels[0].A.shape[0]
    B = np.column_stack([ex["b"].ravel(), np.ones(n), np.zeros(n)])
    for method in METHODS:
        with pytest.raises(ValueError):
            ml.solve_many(B, X0=np.ones((n, 2)), accel=method)
        with pytest.raises(NotImplementedError):
            ml.solve_many(B.astype(complex), accel=method)
        # maxiter=None: min(n, 40) inner iterations, as solve
        _many_equals_per_column(ml, B, tol=1e-12, maxiter=None, accel=method)
        # maxiter > n: solve's warning, raised once per call
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            X, info = ml.solve_many(B, tol=1e-12, maxiter=n + 5, accel=method, return_info=True)
        assert len([w for w in caught if "maximum allowed" in str(w.message)]) == 1
        Xr, ir, _ = _per_column(ml, B, tol=1e-12, maxiter=n + 5, accel=method)
        assert np.array_equal(X, Xr) and list(info) == ir
    with pytest.raises(ValueError):            # AMLI needs fgmres, as in solve
        ml.solve_many(B, accel="gmres", cycle="AMLI")
