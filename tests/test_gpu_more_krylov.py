"""MultilevelSolver.solve / solve_many(accel='cgnr' | 'cgne' | 'minimal_residual' | 'steepest_descent' |
'gmres_householder') on the GPU: the resident drivers amgb_solve_krylov / amgb_solve_many_krylov.

solve reproduces what the real reference's ml.solve(accel=...) computed (tests/golden/krylov_more/): iterate, info,
residual list and warnings.  CUDA tensors give the host result bit for bit, and column j of solve_many is
solve(B[:, j], ...) bit for bit.
"""
import os
import warnings

import numpy as np
import pytest

from conftest import GOLDEN_ALL, GOLDEN_DIR, golden_path
from test_oracle_more_krylov import RUNS, case, check_against_golden, method_of

pytestmark = pytest.mark.gpu
METHODS = ("cgnr", "cgne", "minimal_residual", "steepest_descent")
STOP_WORDS = {("minimal_residual", 1): "Indefinite matrix detected in minimal residual",
              ("steepest_descent", 1): "Indefinite matrix detected in steepest descent"}


def _torch():
    return pytest.importorskip("torch")


def _same(a, b):
    """bit for bit, NaN where NaN"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def _quiet(fn, *a, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with np.errstate(invalid="ignore"):
            return fn(*a, **kw)


def _nonsymmetric():
    """cfg9's upwind advection operator (nonsymmetric) on a hierarchy the batched cycle covers: weighted Jacobi on
    every level instead of AIR's F/C Jacobi."""
    from pyamg_b200.hierarchy_io import load_hierarchy
    from pyamg_b200.relaxation.smoothing import change_smoothers
    ml, ex = load_hierarchy(golden_path("cfg9_air_fcjacobi_advection2d"))
    sm = ("jacobi", {"omega": 2.0 / 3.0})
    change_smoothers(ml, sm, sm)
    return ml, ex


@pytest.mark.parametrize("name", GOLDEN_ALL)
def test_solve_matches_golden(name, load_golden):
    ml, ex = load_golden(name)
    kg = np.load(os.path.join(GOLDEN_DIR, "krylov_more", name + ".npz"))
    for tag in RUNS:
        b, kw = case(tag, ex)
        m = method_of(tag)
        res = []
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            with np.errstate(invalid="ignore"):
                x, info = ml.solve(b, accel=m, residuals=res, return_info=True, **kw)
        check_against_golden(x, info, res, kg, tag)
        if info == -1:
            assert any("detected in" in str(w.message) for w in caught), tag
        else:
            assert not any("detected in" in str(w.message) for w in caught), tag


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg9_air_fcjacobi_advection2d"])
def test_tensors_equal_host(name, method, load_golden):
    torch = _torch()
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    b = ex["b"].ravel()
    x0 = ex["x0"].ravel()
    for kw in (dict(), dict(x0=x0, cycle="W", tol=1e-3, maxiter=20)):
        rh = []
        xh, ih = _quiet(ml.solve, b, accel=method, residuals=rh, return_info=True, tol=kw.get("tol", 1e-10),
                        maxiter=kw.get("maxiter", 8), x0=kw.get("x0"), cycle=kw.get("cycle", "V"))
        x0d = None if "x0" not in kw else torch.tensor(x0, device="cuda")
        x0_copy = None if x0d is None else x0d.clone()
        for bd in (torch.tensor(b, device="cuda"),
                   torch.tensor(np.repeat(b, 2), device="cuda")[::2],               # non-contiguous
                   ):
            rd = []
            xd, idd = _quiet(ml.solve, bd, accel=method, residuals=rd, return_info=True, tol=kw.get("tol", 1e-10),
                             maxiter=kw.get("maxiter", 8), x0=x0d, cycle=kw.get("cycle", "V"))
            assert xd.is_cuda and xd.dtype == torch.float64 and xd.shape == (n,)
            assert _same(xd.cpu().numpy(), xh) and idd == ih and _same(rd, rh)
            if x0d is not None:
                assert torch.equal(x0d, x0_copy)
    # a float32 right-hand side is converted on the device as the host path converts it
    b32 = b.astype(np.float32)
    rh, rd = [], []
    xh, ih = _quiet(ml.solve, b32, accel=method, residuals=rh, return_info=True, tol=1e-8, maxiter=5)
    xd, idd = _quiet(ml.solve, torch.tensor(b32, device="cuda"), accel=method, residuals=rd, return_info=True,
                     tol=1e-8, maxiter=5)
    assert _same(xd.cpu().numpy(), xh) and idd == ih and _same(rd, rh)


def _per_column(ml, B, X0=None, **kw):
    xs, infos, lists = [], [], []
    for j in range(B.shape[1]):
        rj = []
        xj, ij = _quiet(ml.solve, B[:, j], x0=None if X0 is None else X0[:, j].copy(), residuals=rj,
                        return_info=True, **kw)
        xs.append(xj)
        infos.append(ij)
        lists.append(rj)
    return np.column_stack(xs), infos, lists


def _many_equals_per_column(ml, B, X0=None, dev=False, **kw):
    res = []
    if dev:
        torch = _torch()
        Bd = torch.tensor(B, device="cuda")
        X0d = None if X0 is None else torch.tensor(X0, device="cuda")
        Xd, info = _quiet(ml.solve_many, Bd, X0=X0d, residuals=res, return_info=True, **kw)
        assert Xd.is_cuda and tuple(Xd.shape) == B.shape
        X = Xd.cpu().numpy()
    else:
        X, info = _quiet(ml.solve_many, B, X0=X0, residuals=res, return_info=True, **kw)
        assert X.shape == B.shape and X.dtype == np.float64 and X.flags.c_contiguous
    Xr, ir, rr = _per_column(ml, B, X0, **kw)
    assert len(res) == B.shape[1]
    for j in range(B.shape[1]):
        assert info[j] == ir[j], j
        assert _same(X[:, j], Xr[:, j]), j
        assert _same(res[j], rr[j]), j
    return X, info, res


def _block(b, n, k, seed):
    rng = np.random.default_rng(seed)
    cols = [b, np.zeros(n), 1e-6 * b + 1e-9 * rng.standard_normal(n)]
    while len(cols) < k:
        cols.append(rng.standard_normal(n))
    return np.column_stack(cols[:k])


@pytest.mark.parametrize("dev", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("k", [3, 8, 11], ids=["k3", "k8", "k11"])
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "nonsymmetric"])
def test_many_columns_equal_solve(name, method, k, dev, load_golden):
    if dev:
        _torch()
    ml, ex = _nonsymmetric() if name == "nonsymmetric" else load_golden(name)
    n = ml.levels[0].A.shape[0]
    b = ex["b"].ravel()
    B = _block(b, n, k, k)
    X, info, res = _many_equals_per_column(ml, B, dev=dev, tol=1e-4, maxiter=12, accel=method)
    if method != "steepest_descent":
        assert info[1] == 0 and len(res[1]) == 1          # zero column: converged before the loop
    else:
        assert info[1] == 12 and np.isnan(X[:, 1]).all()  # zero column: 0 / 0 on the first step, as the reference
    assert len({len(r) for r in res}) > 1 or len({int(i) for i in info}) > 1
    X0 = np.random.default_rng(k + 1).standard_normal((n, k))
    _many_equals_per_column(ml, B, X0=X0, dev=dev, tol=1e-4, maxiter=10, cycle="W", accel=method)


@pytest.mark.parametrize("method", ["minimal_residual", "steepest_descent"])
def test_indefinite_operator_stops_with_minus_one(method):
    from pyamg_b200.aggregation import smoothed_aggregation_solver
    from pyamg_b200.gallery import poisson
    A = -poisson((40, 40), format="csr")
    ml = smoothed_aggregation_solver(A, max_coarse=20)
    n = A.shape[0]
    B = np.column_stack([np.random.default_rng(s).standard_normal(n) for s in range(3)] + [np.zeros(n)])
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        with np.errstate(invalid="ignore"):
            X, info = ml.solve_many(B, tol=1e-8, maxiter=20, accel=method, return_info=True)
    if method == "steepest_descent":                      # z'Az < 0 on the first step
        assert list(info[:3]) == [-1, -1, -1]
        assert len([w for w in caught if STOP_WORDS[(method, 1)] in str(w.message)]) == 1
    for w in {str(w.message) for w in caught}:
        assert sum(str(c.message) == w for c in caught) == 1          # each distinct warning once
    _many_equals_per_column(ml, B, tol=1e-8, maxiter=20, accel=method)


@pytest.mark.parametrize("method", METHODS)
def test_batched_launches_versus_single(method, load_golden):
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(3).standard_normal((n, 4))
    _quiet(ml.solve, B[:, 0], tol=0, maxiter=3, accel=method)
    single = ml.last_launches()
    _quiet(ml.solve_many, B, tol=0, maxiter=3, accel=method)
    assert ml.last_launches() < 2 * single


def test_krylov_module_functions(load_golden):
    import pyamg_b200.krylov as K
    from scipy.sparse.linalg import aslinearoperator
    ml, ex = load_golden("cfg9_air_fcjacobi_advection2d")
    A = ml.levels[0].A
    b = ex["b"].ravel()
    M = ml.aspreconditioner(cycle="W")
    for m in METHODS + ("gmres_householder",):
        fn = getattr(K, m)
        assert m in K.__all__
        r1, r2 = [], []
        x1, i1 = _quiet(fn, A, b, tol=1e-8, maxiter=6, M=M, residuals=r1)
        x2, i2 = _quiet(ml.solve, b, tol=1e-8, maxiter=6, cycle="W", accel=m, residuals=r2, return_info=True)
        assert _same(x1, x2) and i1 == i2 and _same(r1, r2), m
        with pytest.raises(NotImplementedError):
            fn(A, b, M=M, callback=lambda x: None)
        with pytest.raises(NotImplementedError):
            fn(A, b, M=aslinearoperator(A))
        if m in ("cgnr", "cgne", "steepest_descent"):
            for crit in ("rr+", "MrMr", "rMr"):
                with pytest.raises(NotImplementedError):
                    fn(A, b, M=M, criteria=crit)


@pytest.mark.parametrize("method", ["cgnr", "cgne"])
def test_transpose_follows_change_solve_matrix(method):
    from oracle import krylov_more
    ml, ex = _nonsymmetric()
    b = ex["b"].ravel()
    _quiet(ml.solve, b, tol=1e-8, maxiter=4, accel=method)          # uploads A^H of the first matrix
    A2 = (2.0 * ml.levels[0].A).tocsr()
    ml.change_solve_matrix(A2)
    rg, ro = [], []
    x, info = _quiet(ml.solve, b, tol=1e-10, maxiter=6, accel=method, residuals=rg, return_info=True)
    M = ml.aspreconditioner(cycle="V")
    xo, io = getattr(krylov_more, method)(A2, b, tol=1e-10, maxiter=6, M=lambda r: M @ r, residuals=ro)
    assert info == io and len(rg) == len(ro)
    assert np.allclose(rg, ro, rtol=1e-8)
    assert np.linalg.norm(x - xo) / np.linalg.norm(xo) < 1e-9


def test_maxiter_clamp_and_gmres_householder(load_golden):
    ml, ex = load_golden("cfg2_sa_jacobi_poisson2d")
    n = ml.levels[0].A.shape[0]
    b = ex["b"].ravel()
    for m in ("cgnr", "cgne"):
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            r1 = []
            x1, i1 = ml.solve(b, tol=1e-30, maxiter=2 * n, accel=m, residuals=r1, return_info=True)
        assert len([w for w in caught if "maximum allowed inner iterations" in str(w.message)]) == 1
        r2 = []
        x2, i2 = _quiet(ml.solve, b, tol=1e-30, maxiter=None, accel=m, residuals=r2, return_info=True)
        assert _same(x1, x2) and i1 == i2 and _same(r1, r2) and len(r1) <= int(np.ceil(1.3 * n)) + 3
        B = np.column_stack([b, np.ones(n)])
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            ml.solve_many(B, tol=1e-6, maxiter=2 * n, accel=m)
        assert len([w for w in caught if "maximum allowed inner iterations" in str(w.message)]) == 1
        with pytest.raises(ValueError):
            ml.solve(b, maxiter=0, accel=m)
    for kw in (dict(tol=1e-10, maxiter=12), dict(tol=1e-3, maxiter=25, cycle="W", x0=ex["x0"].ravel())):
        ra, rb = [], []
        xa, ia = _quiet(ml.solve, b, accel="gmres_householder", residuals=ra, return_info=True, **kw)
        xb, ib = _quiet(ml.solve, b, accel="gmres", residuals=rb, return_info=True, **kw)
        assert _same(xa, xb) and ia == ib and _same(ra, rb)
    B = _block(b, n, 3, 1)
    Ra, Rb = [], []
    Xa, Ia = _quiet(ml.solve_many, B, tol=1e-8, maxiter=10, accel="gmres_householder", residuals=Ra, return_info=True)
    Xb, Ib = _quiet(ml.solve_many, B, tol=1e-8, maxiter=10, accel="gmres", residuals=Rb, return_info=True)
    assert _same(Xa, Xb) and list(Ia) == list(Ib) and all(_same(p, q) for p, q in zip(Ra, Rb))
    torch = _torch()
    xd = _quiet(ml.solve, torch.tensor(b, device="cuda"), tol=1e-10, maxiter=12, accel="gmres_householder")
    assert _same(xd.cpu().numpy(), _quiet(ml.solve, b, tol=1e-10, maxiter=12, accel="gmres"))
