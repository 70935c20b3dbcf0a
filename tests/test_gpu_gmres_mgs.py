"""MultilevelSolver.solve / solve_many(accel='gmres_mgs') and pyamg_b200.krylov.gmres_mgs on the GPU: modified
Gram-Schmidt GMRES resident in HBM (amgb_solve_gmres / amgb_solve_many_gmres with AMGB_FLAG_MGS).

solve reproduces what the real reference computed (tests/golden/krylov_mgs/): iterate, info and residual list.  CUDA
tensors give the host result bit for bit, and column j of solve_many is solve(B[:, j], ...) bit for bit.
"""
import ctypes
import os
import sys
import warnings

import numpy as np
import pytest

from conftest import GOLDEN_ALL, GOLDEN_DIR, golden_path, relerr
from test_gpu_more_krylov import _quiet, _same, _torch
from test_oracle_gmres_mgs import RUNS, case

pytestmark = pytest.mark.gpu
WIDTHS = [2, 3, 5, 8, 11]


def _device_bytes(ml):
    from pyamg_b200 import _engine as E
    return int(E.lib().amgb_hierarchy_device_bytes(ml.handle))


def _basis_bytes(n, max_inner, K):
    npad = ((n + 2 + 31) // 32) * 32
    return (max_inner + 1) * npad * K * 8


def _solve(ml, b, reorth=False, cycle="V", **kw):
    """solve(accel='gmres_mgs'), or with reorth pyamg_b200.krylov.gmres_mgs(A, b, M=ml.aspreconditioner(cycle))"""
    res = []
    if reorth:
        import pyamg_b200.krylov as K
        x, info = _quiet(K.gmres_mgs, ml.levels[0].A, b, M=ml.aspreconditioner(cycle=cycle), reorth=True,
                         residuals=res, **kw)
    else:
        x, info = _quiet(ml.solve, b, accel="gmres_mgs", cycle=cycle, residuals=res, return_info=True, **kw)
    return x, info, res


def _oracle(ml, b, reversed_rows=False, **kw):
    """oracle/krylov_mgs.py on the oracle's cycle; reversed_rows: every SpMV sums its row backwards, the rounding-level
    perturbation conftest.summation_order_sensitivity uses as the yardstick"""
    import scipy.sparse as sp
    import oracle
    from oracle.krylov_mgs import run
    cyc = oracle.Cycle(oracle.hierarchy_spec(ml), coarse_pinv=ml.coarse_solver.P)
    orig = oracle.matvec

    def backwards(A, v, kernels="oracle"):
        C = A.tocsr()
        ip = C.indptr
        idx = (np.concatenate([np.arange(ip[i + 1] - 1, ip[i] - 1, -1) for i in range(C.shape[0])])
               if C.nnz else np.zeros(0, dtype=int))
        return orig(sp.csr_array((C.data[idx], C.indices[idx], ip), shape=C.shape), v, kernels)

    if reversed_rows:
        oracle.matvec = backwards
    try:
        res = []
        x, info = _quiet(run, cyc, b, residuals=res, **kw)
    finally:
        oracle.matvec = orig
    return x, info, res


@pytest.mark.parametrize("name", GOLDEN_ALL)
def test_solve_matches_golden(name, load_golden):
    ml, ex = load_golden(name)
    kg = np.load(os.path.join(GOLDEN_DIR, "krylov_mgs", name + ".npz"))
    for tag in RUNS:
        b, kw = case(tag, ex, kg)
        x, info, res = _solve(ml, b, **kw)
        ref_x, ref_res = kg["x_ref_" + tag], kg["residuals_" + tag]
        assert info == int(kg["info_" + tag][0]), tag
        assert len(res) == len(ref_res), tag
        if tag == "mgs_stag":                  # the residuals are rounding noise of b - A x; x moved by ~3e-15
            assert info == -1 and relerr(x, ref_x) < 1e-14, tag
            continue
        assert np.allclose(res, ref_res, rtol=1e-5, atol=1e-12 * res[0]), tag
        xo, _, _ = _oracle(ml, b, **kw)
        xr, _, _ = _oracle(ml, b, reversed_rows=True, **kw)
        scale = np.linalg.norm(kg["x_ref_mgsW"]) if tag == "mgs_zero" else np.linalg.norm(ref_x)
        bound = max(1e-9, 20 * np.linalg.norm(xr - xo) / scale)
        assert np.linalg.norm(x - ref_x) / scale < bound, tag


@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg5_sa_bjacobi_elasticity",
                                  "cfg9_air_fcjacobi_advection2d", "cfg13_rs_gsnr_gsne_advdiff2d"])
def test_oracle_on_fresh_rhs(name, load_golden):
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(17)
    for kw in (dict(tol=1e-8, maxiter=15), dict(tol=1e-6, maxiter=30, cycle="W", x0=rng.standard_normal(n)),
               dict(tol=1e-8, maxiter=4, restart=3), dict(tol=1e-8, maxiter=10, reorth=True)):
        b = rng.standard_normal(n)
        solve_kw = {k: v for k, v in kw.items() if k != "restart"}
        if "restart" in kw:                    # solve has no restart argument: the C entry directly
            from pyamg_b200 import _engine as E
            x, info, res = _c_single(ml, b, kw["restart"], kw["maxiter"], E.FLAG_X0_ZERO | E.FLAG_MGS, kw["tol"])
        else:
            x, info, res = _solve(ml, b, **solve_kw)
        xo, io, ro = _oracle(ml, b, **kw)
        assert info == io and len(res) == len(ro), kw
        assert np.allclose(res, ro, rtol=1e-6, atol=1e-13 * ro[0]), kw
        assert relerr(x, xo) < 1e-9, kw


@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg9_air_fcjacobi_advection2d"])
def test_tensors_equal_host(name, load_golden):
    torch = _torch()
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    b = ex["b"].ravel()
    x0 = ex["x0"].ravel()
    for kw in (dict(tol=1e-10, maxiter=12), dict(x0=x0, cycle="W", tol=1e-3, maxiter=20)):
        xh, ih, rh = _solve(ml, b, **kw)
        x0d = None if "x0" not in kw else torch.tensor(x0, device="cuda")
        x0_copy = None if x0d is None else x0d.clone()
        for bd in (torch.tensor(b, device="cuda"), torch.tensor(np.repeat(b, 2), device="cuda")[::2]):
            xd, idd, rd = _solve(ml, bd, **dict(kw, x0=x0d))
            assert xd.is_cuda and xd.dtype == torch.float64 and xd.shape == (n,)
            assert _same(xd.cpu().numpy(), xh) and idd == ih and _same(rd, rh)
            if x0d is not None:
                assert torch.equal(x0d, x0_copy)
    xh, ih, rh = _solve(ml, b, reorth=True, tol=1e-10, maxiter=12)
    xd, idd, rd = _solve(ml, torch.tensor(b, device="cuda"), reorth=True, tol=1e-10, maxiter=12)
    assert _same(xd.cpu().numpy(), xh) and idd == ih and _same(rd, rh)


def _per_column(ml, B, X0=None, **kw):
    xs, infos, lists = [], [], []
    for j in range(B.shape[1]):
        x, i, r = _solve(ml, B[:, j], x0=None if X0 is None else X0[:, j].copy(), **kw)
        xs.append(x)
        infos.append(i)
        lists.append(r)
    return np.column_stack(xs), infos, lists


def _many_equals_per_column(ml, B, X0=None, dev=False, **kw):
    res = []
    if dev:
        torch = _torch()
        Bd = torch.tensor(B, device="cuda")
        X0d = None if X0 is None else torch.tensor(X0, device="cuda")
        Xd, info = _quiet(ml.solve_many, Bd, X0=X0d, residuals=res, return_info=True, accel="gmres_mgs", **kw)
        assert Xd.is_cuda and tuple(Xd.shape) == B.shape
        X = Xd.cpu().numpy()
    else:
        X, info = _quiet(ml.solve_many, B, X0=X0, residuals=res, return_info=True, accel="gmres_mgs", **kw)
        assert X.shape == B.shape and X.dtype == np.float64 and X.flags.c_contiguous
    nbytes = _device_bytes(ml)
    Xr, ir, rr = _per_column(ml, B, X0, **kw)
    assert len(res) == B.shape[1]
    for j in range(B.shape[1]):
        assert info[j] == ir[j], j
        assert _same(X[:, j], Xr[:, j]), j
        assert _same(res[j], rr[j]), j
    return X, info, res, nbytes


def _block(b, n, k, seed):
    """b, a zero column, b slightly perturbed, a tiny multiple of b, then random columns"""
    rng = np.random.default_rng(seed)
    cols = [b, np.zeros(n), b + 1e-3 * rng.standard_normal(n), 1e-8 * b]
    while len(cols) < k:
        cols.append(rng.standard_normal(n))
    return np.column_stack(cols[:k])


@pytest.mark.parametrize("dev", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("k", WIDTHS, ids=[f"k{k}" for k in WIDTHS])
@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg5_sa_bjacobi_elasticity"])
def test_many_columns_equal_solve(name, k, dev):
    from pyamg_b200.hierarchy_io import load_hierarchy
    if dev:
        _torch()
    ml, ex = load_hierarchy(golden_path(name))            # fresh: the first batched call allocates the basis store
    n = ml.levels[0].A.shape[0]
    b = ex["b"].ravel()
    B = _block(b, n, k, k)
    before = _device_bytes(ml)
    X, info, res, nbytes = _many_equals_per_column(ml, B, dev=dev, tol=1e-6, maxiter=30)
    assert nbytes - before >= _basis_bytes(n, 30, 2)      # the batched path ran: its basis store is counted
    assert info[1] == 0 and len(res[1]) == 1 and not X[:, 1].any()   # zero column: converged before the loop
    if k >= 4:
        assert len({len(r) for r in res}) > 1             # columns left the inner loop at different iterations
    X0 = np.random.default_rng(k + 1).standard_normal((n, k))
    _many_equals_per_column(ml, B, X0=X0, dev=dev, tol=1e-4, maxiter=10, cycle="W")


def test_batched_launches_versus_single(load_golden):
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(3).standard_normal((n, 4))
    _quiet(ml.solve, B[:, 0], tol=0, maxiter=6, accel="gmres_mgs")
    single = ml.last_launches()
    _quiet(ml.solve_many, B, tol=0, maxiter=6, accel="gmres_mgs")
    assert 0 < ml.last_launches() < 2 * single


def _c_single(ml, b, restart, maxiter, flags, tol, rows=64):
    from pyamg_b200 import _engine as E
    n = b.size
    bh = np.ascontiguousarray(b, dtype=np.float64)
    x = np.zeros(n)
    r = np.zeros(rows)
    nr, inf = ctypes.c_int32(0), ctypes.c_int32(0)
    E.check(E.lib().amgb_solve_gmres(ml.handle, bh.ctypes.data, x.ctypes.data, tol, restart, maxiter, E.CYCLES["V"],
                                     flags, E.f64p(r), rows, ctypes.byref(nr), ctypes.byref(inf)))
    return x, inf.value, list(r[:min(nr.value, rows)])


@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg6_rs_gsfwd_none_poisson3d"])
def test_restarts_and_reorth_through_the_c_abi(name, load_golden):
    from pyamg_b200 import _engine as E
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    B = _block(ex["b"].ravel(), n, 5, 2)
    rows = 64
    for flags in (E.FLAG_X0_ZERO | E.FLAG_MGS, E.FLAG_X0_ZERO | E.FLAG_MGS | E.FLAG_REORTH):
        X = np.zeros((n, 5))
        res = np.zeros((rows, 5))
        nres, info = np.zeros(5, dtype=np.int32), np.zeros(5, dtype=np.int32)
        E.check(E.lib().amgb_solve_many_gmres(ml.handle, 5, np.ascontiguousarray(B).ctypes.data, X.ctypes.data, 1e-12,
                                              3, 4, E.CYCLES["V"], flags, E.f64p(res), rows, E.i32p(nres),
                                              E.i32p(info)))
        for j in range(5):
            x, i, r = _c_single(ml, B[:, j], 3, 4, flags, 1e-12, rows)
            assert info[j] == i and _same(X[:, j], x) and _same(res[:len(r), j], r), j
        assert nres[0] > 4                                 # more than one outer iteration ran


def test_reorth_pass_on_an_exhausted_krylov_space():
    """n = 16 with maxiter = n: the last new vector lies in the Krylov space already, its norm collapses and
    reorth=True takes the second pass; batched columns still equal single solves, and the result solves A x = b."""
    from pyamg_b200 import _engine as E
    from pyamg_b200.classical import ruge_stuben_solver
    from pyamg_b200.gallery import poisson
    A = poisson((4, 4), format="csr")
    ml = ruge_stuben_solver(A, max_coarse=4)
    n = A.shape[0]
    B = np.random.default_rng(4).standard_normal((n, 3))
    flags = E.FLAG_X0_ZERO | E.FLAG_MGS | E.FLAG_REORTH
    X = np.zeros((n, 3))
    info = np.zeros(3, dtype=np.int32)
    res = np.zeros((n + 3, 3))
    nres = np.zeros(3, dtype=np.int32)
    E.check(E.lib().amgb_solve_many_gmres(ml.handle, 3, np.ascontiguousarray(B).ctypes.data, X.ctypes.data, 0.0, 0, n,
                                          E.CYCLES["V"], flags, E.f64p(res), n + 3, E.i32p(nres), E.i32p(info)))
    for j in range(3):
        x, i, r = _c_single(ml, B[:, j], 0, n, flags, 0.0, n + 3)
        assert info[j] == i and _same(X[:, j], x), j
        assert np.linalg.norm(A @ x - B[:, j]) < 1e-8 * np.linalg.norm(B[:, j]), j
        xo, io, _ = _oracle(ml, B[:, j], tol=0.0, maxiter=n, reorth=True)
        assert relerr(x, xo) < 1e-8, j


def test_basis_store_narrows_to_what_fits():
    """Poisson 100^3 with maxiter=1500: eight columns would need about 96 GB of basis vectors, more than the card
    holds, so the call runs at a narrower width -- with every column still equal to its single solve."""
    from pyamg_b200.classical import ruge_stuben_solver
    from pyamg_b200.gallery import poisson
    A = poisson((100, 100, 100), format="csr")
    ml = ruge_stuben_solver(A, max_coarse=500)
    n = A.shape[0]
    B = np.random.default_rng(8).standard_normal((n, 8))
    before = _device_bytes(ml)
    X, info, res, nbytes = _many_equals_per_column(ml, B, tol=1e-8, maxiter=1500)
    assert (info == 0).all()
    assert nbytes - before < _basis_bytes(n, 1500, 8)             # the 8-wide store was never kept
    assert nbytes - before >= _basis_bytes(n, 1500, 2)
    x, i1 = ml.solve(B[:, 0], tol=1e-8, maxiter=50, return_info=True)     # the hierarchy stays usable
    assert i1 == 0


def test_maxiter_clamp_and_defaults(load_golden):
    from pyamg_b200.classical import ruge_stuben_solver
    from pyamg_b200.gallery import poisson
    A = poisson((6, 6), format="csr")
    ml = ruge_stuben_solver(A, max_coarse=10)
    n = A.shape[0]
    b = np.random.default_rng(1).standard_normal(n)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        r1 = []
        x1, i1 = ml.solve(b, tol=1e-30, maxiter=n + 5, accel="gmres_mgs", residuals=r1, return_info=True)
    assert len([w for w in caught if "Setting maxiter to maximum allowed, n." in str(w.message)]) == 1
    x2, i2, r2 = _solve(ml, b, tol=1e-30, maxiter=n)
    assert _same(x1, x2) and i1 == i2 and _same(r1, r2)
    x3, i3, r3 = _solve(ml, b, tol=1e-30, maxiter=None)           # min(n, 40) = n here
    assert _same(x1, x3) and i1 == i3 and _same(r1, r3)
    B = np.column_stack([b, np.ones(n), np.zeros(n)])
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        X, info = ml.solve_many(B, tol=1e-12, maxiter=n + 5, accel="gmres_mgs", return_info=True)
    assert len([w for w in caught if "maximum allowed" in str(w.message)]) == 1
    Xr, ir, _ = _per_column(ml, B, tol=1e-12, maxiter=n + 5)
    assert _same(X, Xr) and list(info) == ir
    ml2, ex = load_golden("cfg2_sa_jacobi_poisson2d")
    with pytest.raises(ValueError):                                # AMLI needs fgmres, as in solve
        ml2.solve(ex["b"], accel="gmres_mgs", cycle="AMLI")
    with pytest.raises(ValueError):
        ml2.solve_many(np.column_stack([ex["b"].ravel()] * 2), accel="gmres_mgs", cycle="AMLI")


def test_krylov_module_functions(load_golden):
    import pyamg_b200.krylov as K
    from scipy.sparse.linalg import aslinearoperator
    ml, ex = load_golden("cfg9_air_fcjacobi_advection2d")
    A = ml.levels[0].A
    b = ex["b"].ravel()
    M = ml.aspreconditioner(cycle="W")
    assert "gmres_mgs" in K.__all__
    r0 = []
    x0, i0 = _quiet(ml.solve, b, tol=1e-8, maxiter=6, cycle="W", accel="gmres_mgs", residuals=r0, return_info=True)
    for fn in (K.gmres_mgs, lambda *a, **kw: K.gmres(*a, orthog="mgs", **kw)):
        r1 = []
        x1, i1 = _quiet(fn, A, b, tol=1e-8, maxiter=6, M=M, residuals=r1)
        assert _same(x1, x0) and i1 == i0 and _same(r1, r0)
        with pytest.raises(NotImplementedError):
            fn(A, b, M=M, callback=lambda x: None)
        with pytest.raises(NotImplementedError):
            fn(A, b, M=M, restart=5)
        with pytest.raises(NotImplementedError):
            fn(A, b, M=aslinearoperator(A))
    with pytest.raises(NotImplementedError):
        K.gmres_mgs(A, b, M=M, restrt=5)
    with pytest.raises(NotImplementedError):
        K.gmres(A, b, M=M, orthog="cgs")


def test_flag_validation(load_golden):
    from pyamg_b200 import _engine as E
    ml, ex = load_golden("cfg2_sa_jacobi_poisson2d")
    n = ml.levels[0].A.shape[0]
    b = np.ascontiguousarray(ex["b"].ravel())
    B = np.ascontiguousarray(np.column_stack([b, b]))
    L = E.lib()
    for flags in (E.FLAG_MGS | E.FLAG_FLEXIBLE, E.FLAG_REORTH, E.FLAG_REORTH | E.FLAG_FLEXIBLE):
        x = np.zeros(n)
        nr, inf = ctypes.c_int32(0), ctypes.c_int32(0)
        r = np.zeros(8)
        assert L.amgb_solve_gmres(ml.handle, b.ctypes.data, x.ctypes.data, 1e-8, 0, 5, E.CYCLES["V"], flags,
                                  E.f64p(r), 8, ctypes.byref(nr), ctypes.byref(inf)) == E.EINVAL
        X = np.zeros((n, 2))
        R = np.zeros((8, 2))
        nres, info = np.zeros(2, dtype=np.int32), np.zeros(2, dtype=np.int32)
        assert L.amgb_solve_many_gmres(ml.handle, 2, B.ctypes.data, X.ctypes.data, 1e-8, 0, 5, E.CYCLES["V"], flags,
                                       E.f64p(R), 8, E.i32p(nres), E.i32p(info)) == E.EINVAL
    x, i, res = _solve(ml, b, tol=1e-8, maxiter=5)                 # the hierarchy stays usable
    assert len(res) > 1


def test_resident_without_the_reference_or_host_cycles(load_golden, monkeypatch):
    """The calls run inside the engine: no import of the reference, and no host cycle (amgb_solve / amgb_solve_ex,
    what aspreconditioner() would call once per application)."""
    import pyamg_b200.krylov as K
    from pyamg_b200 import _engine as E
    torch = _torch()
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    b = ex["b"].ravel()
    monkeypatch.setattr(sys, "path", [p for p in sys.path if "_ref" not in p])
    for mod in [m for m in sys.modules if m == "pyamg" or m.startswith("pyamg.")]:
        monkeypatch.delitem(sys.modules, mod)
    L = E.lib()

    def refuse(*a, **kw):
        raise AssertionError("a host cycle ran")

    monkeypatch.setattr(L, "amgb_solve_ex", refuse)
    monkeypatch.setattr(L, "amgb_solve", refuse)
    M = ml.aspreconditioner()
    x1, i1, _ = _solve(ml, b, tol=1e-8, maxiter=20)
    assert ml.last_launches() > 0
    xd, idd, _ = _solve(ml, torch.tensor(b, device="cuda"), tol=1e-8, maxiter=20)
    X, info = _quiet(ml.solve_many, np.column_stack([b, 2 * b]), tol=1e-8, maxiter=20, accel="gmres_mgs",
                     return_info=True)
    xk, ik = _quiet(K.gmres, ml.levels[0].A, b, M=M, tol=1e-8, maxiter=20, orthog="mgs")
    assert i1 == 0 and idd == 0 and list(info) == [0, 0] and ik == 0
    assert _same(xd.cpu().numpy(), x1) and _same(X[:, 0], x1) and _same(xk, x1)
    assert not any(m == "pyamg" or m.startswith("pyamg.") for m in sys.modules)


@pytest.mark.parametrize("env", [{"AMGB_NO_PERMUTE": "1"}, {"AMGB_NO_GRAPH": "1"}, {"AMGB_NO_TILES": "1"},
                                 {"AMGB_TILE_MIN_NNZ": "0"}])
@pytest.mark.parametrize("name", ["cfg3_rs_mcgs_poisson3d", "cfg5_sa_bjacobi_elasticity"])
def test_kernel_paths(name, env, monkeypatch):
    from pyamg_b200.hierarchy_io import load_hierarchy
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ml, ex = load_hierarchy(golden_path(name))
    kg = np.load(os.path.join(GOLDEN_DIR, "krylov_mgs", name + ".npz"))
    b, kw = case("mgs", ex, kg)
    x, info, res = _solve(ml, b, **kw)
    assert info == int(kg["info_mgs"][0]) and len(res) == len(kg["residuals_mgs"])
    assert np.allclose(res, kg["residuals_mgs"], rtol=1e-5, atol=1e-12 * res[0])
    n = ml.levels[0].A.shape[0]
    B = _block(ex["b"].ravel(), n, 3, 9)
    _many_equals_per_column(ml, B, tol=1e-10, maxiter=12)
