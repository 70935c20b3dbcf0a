"""CPU tests of which engine entry solve, solve_many and pyamg_b200.krylov call, with which scalar arguments and
residual buffers, and which warnings and exceptions they raise around the call.

The engine library is replaced by a recording fake: no GPU, no nvcc and no build.  The fake writes x = x0 + b
(x = b from a zero start) and chosen info, reason and residual counts through the pointers it is given, so the
values handed back to the caller are pinned too."""
import ctypes
import sys
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

import pyamg_b200
from pyamg_b200 import _engine as E
from pyamg_b200 import krylov
from pyamg_b200.hierarchy_io import load_hierarchy
from conftest import golden_path

# argument names of the solve entries; "*" marks a pointer, h / b / x / B / X are not recorded
_SIGS = {
    "amgb_solve": "h b x tol maxiter cycle cycles_per_level *res *nres *info",
    "amgb_solve_ex": "h b x tol maxiter cycle cycles_per_level flags *res *nres *info",
    "amgb_solve_cg": "h b x tol maxiter cycle flags *res *nres *info",
    "amgb_solve_bicgstab": "h b x tol maxiter cycle flags *res *nres *info",
    "amgb_solve_gmres": "h b x tol restart maxiter cycle flags *res max_residuals *nres *info",
    "amgb_solve_krylov": "h method b x tol maxiter cycle flags *res *nres *info *reason",
    "amgb_solve_many": "h k B X tol maxiter cycle cycles_per_level flags *res *nres *info",
    "amgb_solve_many_cg": "h k B X tol maxiter cycle flags *res *nres *info",
    "amgb_solve_many_bicgstab": "h k B X tol maxiter cycle flags *res *nres *info",
    "amgb_solve_many_gmres": "h k B X tol restart maxiter cycle flags *res max_residuals *nres *info",
    "amgb_solve_many_krylov": "h method k B X tol maxiter cycle flags *res *nres *info *reason",
}


class FakeEngine:
    """Stands in for libpyamg_b200.so.  ``calls`` holds (entry, scalar arguments, residual buffer size or None) per
    solve call; amgb_solve is recorded as the amgb_solve_ex call with flags = 0 that it is."""

    def __init__(self):
        self.calls = []
        self.notimpl = set()          # entries that answer ENOTIMPL
        self.info, self.reason, self.nres = 0, 0, 2   # written per column (a scalar, or one value per column)
        self.n = 0

    def __getattr__(self, name):
        if name in _SIGS:
            return lambda *args: self._solve(name, args)
        if name == "amgb_hierarchy_create":
            return self._create
        if name == "amgb_device_count":
            return lambda: 1
        if name == "amgb_last_error":
            return lambda: b"fake engine"
        if name == "amgb_hierarchy_set_transpose0":
            return lambda h, M: self.calls.append((name, {}, None)) or 0
        if name.startswith("amgb_"):
            return lambda *args: 0
        raise AttributeError(name)

    @staticmethod
    def _create(device, ph):
        ph._obj.value = 1
        return 0

    def _column_values(self, v, k):
        return np.broadcast_to(np.asarray(v, dtype=np.int32), (k,))

    def _solve(self, name, args):
        names = _SIGS[name].split()
        a = dict(zip(names, args))
        scalars = {key: v for key, v in a.items() if key not in ("h", "b", "x", "B", "X") and key[0] != "*"}
        if name == "amgb_solve":
            name, scalars = "amgb_solve_ex", dict(scalars, flags=0)
        res = a["*res"]
        rarr = None if res is None else res._arr
        self.calls.append((name, scalars, None if rarr is None else rarr.size))
        if name in self.notimpl:
            return E.ENOTIMPL
        k = a.get("k", 1)
        size = self.n * k
        b = np.ctypeslib.as_array((ctypes.c_double * size).from_address(a.get("b", a.get("B"))))
        x = np.ctypeslib.as_array((ctypes.c_double * size).from_address(a.get("x", a.get("X"))))
        if scalars["flags"] & E.FLAG_X0_ZERO:
            x[:] = 0.0
        x += b
        if rarr is not None:
            rarr.flat[:] = 1.0 / np.arange(1, rarr.size + 1)
        for key, v in (("*nres", self.nres), ("*info", self.info), ("*reason", self.reason)):
            if key in a:
                vals = self._column_values(v, k)
                if hasattr(a[key], "_obj"):
                    a[key]._obj.value = int(vals[0])
                else:
                    a[key]._arr[:] = vals
        return E.OK


@pytest.fixture
def fake(monkeypatch):
    f = FakeEngine()
    monkeypatch.setattr(E, "_lib", f)
    monkeypatch.setitem(sys.modules, "pyamg", None)      # host fallbacks resolve names in scipy.sparse.linalg
    return f


@pytest.fixture
def load(fake):
    made = []

    def _load(name):
        ml = load_hierarchy(golden_path(name))[0]
        fake.n = ml.levels[0].A.shape[0]
        made.append(ml)
        return ml

    def _one_by_one():
        lvl = pyamg_b200.MultilevelSolver.Level()
        lvl.A = sp.csr_matrix(np.array([[2.0]]))
        ml = pyamg_b200.MultilevelSolver([lvl])
        fake.n = 1
        made.append(ml)
        return ml

    _load.one_by_one = _one_by_one
    yield _load
    for ml in made:
        ml._invalidate()             # while the fake is still installed


CFG2 = "cfg2_sa_jacobi_poisson2d"     # n = 1600, symmetric smoothing
CFG9 = "cfg9_air_fcjacobi_advection2d"  # n = 841, non-symmetric smoothing
N = 1600
ACCELS = ["cg", "bicgstab", "gmres", "gmres_householder", "gmres_mgs", "fgmres", "cgnr", "cgne", "minimal_residual",
          "steepest_descent"]
GMRES = ("gmres", "gmres_householder", "gmres_mgs", "fgmres")
SYM_WARNING = ("Incompatible non-symmetric multigrid preconditioner detected, due to presmoother/postsmoother "
               "combination. CG requires SPD preconditioner, not just SPD matrix.")
CG_STOP = "\nIndefinite matrix or preconditioner detected in CG, aborting\n"
GMRES_CLAMP = "Setting maxiter to maximum allowed, n."
CGN_CLAMP = {"cgnr": "maximum allowed inner iterations (maxiter) are the 130% times               the number of dofs",
             "cgne": "maximum allowed inner iterations (maxiter) are the 130% timesthe number of dofs"}


def expected_call(accel, maxiter, n, k=None):
    """(entry, scalars, residual buffer size) the reference's defaults and clamps give for one resident call."""
    many = "_many" if k is not None else ""
    flags = E.FLAG_X0_ZERO
    if accel in GMRES:
        max_inner = min(n, 40) if maxiter is None else min(maxiter, n)
        flags |= (E.FLAG_FLEXIBLE if accel == "fgmres" else 0) | (E.FLAG_MGS if accel == "gmres_mgs" else 0)
        s = dict(tol=1e-7, restart=0, maxiter=0 if maxiter is None else maxiter, cycle=E.CYCLES["W"], flags=flags,
                 max_residuals=max_inner + 3)
        entry, size = f"amgb_solve{many}_gmres", max_inner + 3
    else:
        if accel in ("cg", "bicgstab"):
            its = maxiter if maxiter is not None else (int(1.3 * n) + 2 if accel == "cg" else n + 5)
            entry, s = f"amgb_solve{many}_{accel}", {}
        else:
            cap = int(np.ceil(1.3 * n)) + 2
            if accel in CGN_CLAMP:
                its = cap if maxiter is None or maxiter > 1.3 * n else maxiter
            else:
                its = maxiter if maxiter is not None else (int(1.3 * n) + 2 if accel == "minimal_residual" else n)
            entry, s = f"amgb_solve{many}_krylov", {"method": E.KRYLOV[accel]}
        s.update(tol=1e-7, maxiter=its, cycle=E.CYCLES["W"], flags=flags)
        size = its + 1
    if k is not None:
        s["k"] = k
        size *= k
    return entry, s, size


def _run(fn):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        out = fn()
    return out, [str(w.message) for w in caught]


@pytest.mark.parametrize("maxiter", [None, 3, 2500, 0])
@pytest.mark.parametrize("accel", ACCELS)
def test_solve_calls_the_resident_entry(load, fake, accel, maxiter):
    ml = load(CFG2)
    b = np.ones(N)
    res = []
    if maxiter == 0 and accel not in GMRES:
        with pytest.raises(ValueError, match="Number of iterations must be positive"):
            ml.solve(b, tol=1e-7, maxiter=maxiter, cycle="W", accel=accel, residuals=res)
        assert fake.calls == []
        return
    (x, info), caught = _run(lambda: ml.solve(b, tol=1e-7, maxiter=maxiter, cycle="W", accel=accel, residuals=res,
                                              return_info=True))
    pre = [("amgb_hierarchy_set_transpose0", {}, None)] if accel in CGN_CLAMP else []
    assert fake.calls == pre + [expected_call(accel, maxiter, N)]
    assert isinstance(x, np.ndarray) and x.shape == (N,) and np.array_equal(x, b)
    assert info == 0 and res == [1.0, 0.5]
    want = []
    if maxiter == 2500 and accel in GMRES:
        want = [GMRES_CLAMP]
    if maxiter == 2500 and accel in CGN_CLAMP:
        want = [CGN_CLAMP[accel]]
    assert caught == want


@pytest.mark.parametrize("k", [1, 3, 9])
@pytest.mark.parametrize("maxiter", [None, 3, 2500, 0])
@pytest.mark.parametrize("accel", ACCELS)
def test_solve_many_calls_the_resident_entry(load, fake, accel, maxiter, k):
    ml = load(CFG2)
    B = np.arange(1.0, N * k + 1).reshape(N, k)
    X0 = np.full((N, k), 0.5)
    res = []
    if maxiter == 0 and accel not in GMRES:
        with pytest.raises(ValueError, match="Number of iterations must be positive"):
            ml.solve_many(B, X0, tol=1e-7, maxiter=maxiter, cycle="W", accel=accel, residuals=res)
        assert fake.calls == []
        return
    (X, info), caught = _run(lambda: ml.solve_many(B, X0, tol=1e-7, maxiter=maxiter, cycle="W", accel=accel,
                                                   residuals=res, return_info=True))
    entry, s, size = expected_call(accel, maxiter, N, None if k == 1 else k)     # k = 1 goes through solve
    pre = [("amgb_hierarchy_set_transpose0", {}, None)] if accel in CGN_CLAMP else []
    assert fake.calls == pre + [(entry, dict(s, flags=s["flags"] & ~E.FLAG_X0_ZERO), size)]
    assert X.shape == (N, k) and X.dtype == np.float64 and np.array_equal(X, B + 0.5)
    assert info.dtype == int and list(info) == [0] * k
    assert res == [[1.0 / (j + 1), 1.0 / (k + j + 1)] for j in range(k)]      # column j of the (rows, k) buffer
    want = []
    if maxiter == 2500 and accel in GMRES:
        want = [GMRES_CLAMP]
    if maxiter == 2500 and accel in CGN_CLAMP:
        want = [CGN_CLAMP[accel]]
    assert caught == want


@pytest.mark.parametrize("accel", ACCELS)
def test_batched_residual_lists_are_columns(load, fake, accel):
    ml = load(CFG2)
    fake.nres = [1, 2, 3]
    res = []
    ml.solve_many(np.ones((N, 3)), tol=1e-7, maxiter=3, cycle="W", accel=accel, residuals=res)
    flat = 1.0 / np.arange(1, fake.calls[-1][2] + 1)
    assert res == [list(flat.reshape(-1, 3)[:j + 1, j]) for j in range(3)]
    fake.calls.clear()
    ml.solve_many(np.ones((N, 3)), tol=1e-7, maxiter=3, cycle="W", accel=accel)
    assert fake.calls[-1][2] == (18 if accel in GMRES else None)      # GMRES always keeps its residual buffer


def test_plain_cycling_entries(load, fake):
    ml = load(CFG2)
    res = []
    x = ml.solve(np.ones((N, 1)), tol=1e-6, maxiter=7, cycle="F", cycles_per_level=2, residuals=res)
    assert x.shape == (N,) and res == [1.0, 0.5]
    call = dict(tol=1e-6, maxiter=7, cycle=E.CYCLES["F"], cycles_per_level=2, flags=E.FLAG_X0_ZERO)
    assert fake.calls == [("amgb_solve_ex", call, 8)]
    fake.calls.clear()
    ml.solve_many(np.ones((N, 3)), tol=1e-6, maxiter=7, cycle="F", cycles_per_level=2)
    assert fake.calls == [("amgb_solve_many", dict(call, k=3), 24)]
    fake.calls.clear()
    fake.notimpl = {"amgb_solve_many"}
    X, info = ml.solve_many(np.ones((N, 3)), np.zeros((N, 3)), maxiter=7, return_info=True)
    assert fake.calls[0][0] == "amgb_solve_many" and fake.calls[0][1]["flags"] == 0
    assert fake.calls[1:] == [("amgb_solve_ex", dict(call, tol=1e-5, cycle=0, cycles_per_level=1, flags=0), 8)] * 3
    assert np.array_equal(X, np.ones((N, 3))) and list(info) == [0, 0, 0]
    fake.calls.clear()
    ml.solve_many(np.ones((N, 1)), maxiter=2)
    assert [c[0] for c in fake.calls] == ["amgb_solve_ex"]
    with pytest.raises(ValueError, match="maxiter must be at least 1"):
        ml.solve_many(np.ones((N, 2)), maxiter=0)
    with pytest.raises(TypeError, match=r"Unrecognized cycle type \(Q\)"):
        ml.solve_many(np.ones((N, 2)), cycle="q")
    with pytest.raises(TypeError, match=r"Unrecognized cycle type \(Q\)"):
        ml.solve_many(np.ones((N, 2)), cycle="q", accel="cg")


def test_callback_loop_calls_one_cycle_at_a_time(load, fake):
    ml = load(CFG2)
    seen, res = [], []
    x, info = ml.solve(np.ones(N), x0=np.full(N, 2.0), maxiter=3, callback=lambda xk: seen.append(xk.copy()),
                       residuals=res, return_info=True)
    one = dict(tol=0.0, maxiter=1, cycle=0, cycles_per_level=1, flags=0)
    assert fake.calls == [("amgb_solve_ex", one, 2)] * 3
    assert [float(s[0]) for s in seen] == [3.0, 4.0, 5.0] and info == 3 and res == [1.0, 0.5, 0.5, 0.5]


@pytest.mark.parametrize("accel", ACCELS)
def test_callback_runs_a_host_solver(load, fake, accel):
    """cg runs the CG host solver; other names are looked up in scipy.sparse.linalg (pyamg is hidden here)."""
    ml = load(CFG2)
    if accel not in ("cg", "bicgstab", "gmres"):
        with pytest.raises(NotImplementedError, match=f"accel='{accel}': GPU-resident accelerators are"):
            ml.solve(np.ones(N), maxiter=2, accel=accel, callback=lambda xk: None)
        assert fake.calls == []
        return
    _run(lambda: ml.solve(np.ones(N), maxiter=2, accel=accel, callback=lambda xk: None))
    assert fake.calls and all(c[0] == "amgb_solve_ex" and c[1]["maxiter"] == 1 for c in fake.calls)


@pytest.mark.parametrize("accel", ACCELS)
def test_one_unknown(load, fake, accel):
    ml = load.one_by_one()
    resident = accel not in GMRES and accel != "bicgstab"
    if accel in ("gmres_householder", "gmres_mgs", "fgmres"):       # no host solver of that name in SciPy
        with pytest.raises(NotImplementedError, match=f"accel='{accel}': GPU-resident accelerators are"):
            ml.solve(np.ones(1), maxiter=3, accel=accel)
        assert fake.calls == []
        if accel == "gmres_householder":       # solve_many's columns run it as 'gmres': SciPy's GMRES
            _run(lambda: ml.solve_many(np.ones((1, 3)), maxiter=3, accel=accel))
            assert {c[0] for c in fake.calls} == {"amgb_solve_ex"}
        else:
            with pytest.raises(NotImplementedError, match=f"accel='{accel}': GPU-resident accelerators are"):
                _run(lambda: ml.solve_many(np.ones((1, 3)), maxiter=3, accel=accel))
        return
    _run(lambda: ml.solve(np.ones(1), maxiter=3, accel=accel))
    names = [c[0] for c in fake.calls]
    if resident:
        assert names[-1] in ("amgb_solve_cg", "amgb_solve_krylov")
    else:
        assert set(names) <= {"amgb_solve_ex"}
    fake.calls.clear()
    _run(lambda: ml.solve_many(np.ones((1, 3)), maxiter=3, accel=accel))
    names = [c[0] for c in fake.calls]
    if resident:
        assert names[-1] in ("amgb_solve_many_cg", "amgb_solve_many_krylov") and len(names) <= 2
    else:
        assert set(names) <= {"amgb_solve_ex"}


@pytest.mark.parametrize("accel", ACCELS)
def test_amli(load, fake, accel):
    ml = load(CFG2)
    if accel != "fgmres":
        with pytest.raises(ValueError, match="AMLI cycles require acceleration"):
            ml.solve(np.ones(N), cycle="AMLI", accel=accel)
        with pytest.raises(ValueError, match="AMLI cycles require acceleration"):
            ml.solve_many(np.ones((N, 3)), cycle="AMLI", accel=accel)
        assert fake.calls == []
        return
    ml.solve(np.ones(N), cycle="AMLI", accel=accel, maxiter=5)
    assert fake.calls == [("amgb_solve_gmres", dict(tol=1e-5, restart=0, maxiter=5, cycle=E.CYCLES["AMLI"],
                                                     flags=E.FLAG_X0_ZERO | E.FLAG_FLEXIBLE, max_residuals=8), 8)]
    fake.calls.clear()
    ml.solve_many(np.ones((N, 3)), cycle="AMLI", accel=accel, maxiter=5)
    assert [c[0] for c in fake.calls] == ["amgb_solve_gmres"] * 3          # column by column


def test_complex_and_out(load, fake):
    ml = load(CFG2)
    bc = np.ones(N) + 1j
    # the CG host solver casts b to float64 (today's behaviour)
    (x, info), caught = _run(lambda: ml.solve(bc, maxiter=2, accel="cg", return_info=True))
    assert x.dtype == np.float64 and {c[0] for c in fake.calls} == {"amgb_solve_ex"}
    for accel in ACCELS[1:]:
        # bicgstab and gmres reach SciPy's solver, whose preconditioner refuses complex vectors
        text = "complex systems are outside" if accel in ("bicgstab", "gmres") else "GPU-resident accelerators are"
        with pytest.raises(NotImplementedError, match=text):
            _run(lambda: ml.solve(bc, maxiter=2, accel=accel))
    with pytest.raises(NotImplementedError, match="complex systems are outside the fp64 hot path"):
        ml.solve_many(np.ones((N, 3)) + 1j, accel="cg")
    with pytest.raises(NotImplementedError, match="complex systems are outside the fp64 hot path"):
        ml.solve_many(np.ones((N, 3)) + 1j)
    with pytest.raises(ValueError, match="out= is supported for plain cycling only"):
        ml.solve(np.ones(N), accel="cg", out=np.empty(N))
    with pytest.raises(ValueError, match="b / x0 have invalid dimensions"):
        ml.solve(np.ones(N + 1), accel="gmres")
    with pytest.raises(NotImplementedError, match="accel='nosuch': GPU-resident accelerators are 'cg', 'bicgstab', "
                                                  "'gmres', 'gmres_householder', 'gmres_mgs', 'fgmres', 'cgnr', "
                                                  "'cgne', 'minimal_residual' and 'steepest_descent'; other names "
                                                  "need pyamg.krylov or scipy.sparse.linalg to provide a host "
                                                  "solver of that name"):
        ml.solve(np.ones(N), accel="nosuch")


def test_cg_symmetric_smoothing_warning_and_stop(load, fake):
    ml = load(CFG9)
    fake.info = -1
    (x, info), caught = _run(lambda: ml.solve(np.ones(841), accel="cg", return_info=True))
    assert info == -1 and caught == [SYM_WARNING, CG_STOP]
    (x, info), caught = _run(lambda: ml.solve(np.ones(841), accel="bicgstab", return_info=True))
    assert info == -1 and caught == [CG_STOP]
    fake.info = [0, -1, -1]
    (X, info), caught = _run(lambda: ml.solve_many(np.ones((841, 3)), accel="cg", return_info=True))
    assert list(info) == [0, -1, -1] and caught == [SYM_WARNING, CG_STOP]
    fake.info = 0
    _, caught = _run(lambda: ml.solve_many(np.ones((841, 3)), accel="bicgstab"))
    assert caught == []
    fake.info = -1
    _, caught = _run(lambda: ml.solve(np.ones(841), accel="gmres"))
    assert caught == []


STOPS = [("minimal_residual", E.REASON_INDEFINITE_MATRIX, "\nIndefinite matrix detected in minimal residual, stopping.\n"),
         ("steepest_descent", E.REASON_INDEFINITE_MATRIX, "\nIndefinite matrix detected in steepest descent, aborting\n"),
         ("steepest_descent", E.REASON_INDEFINITE_PRECONDITIONER,
          "\nIndefinite preconditioner detected in steepest descent, stopping.\n"),
         ("steepest_descent", E.REASON_SINGULAR_PRECONDITIONER,
          "\nSingular preconditioner detected in steepest descent, stopping.\n")]


@pytest.mark.parametrize("accel,reason,text", STOPS)
def test_krylov_stop_warnings(load, fake, accel, reason, text):
    ml = load(CFG2)
    fake.info, fake.reason = -1, reason
    (x, info), caught = _run(lambda: ml.solve(np.ones(N), accel=accel, return_info=True))
    assert info == -1 and caught == [text]
    fake.info, fake.reason = [-1, 0, -1], [reason, 0, reason]
    (X, info), caught = _run(lambda: ml.solve_many(np.ones((N, 3)), accel=accel, return_info=True))
    assert list(info) == [-1, 0, -1] and caught == [text]


def test_krylov_stop_warnings_by_reason_in_order(load, fake):
    ml = load(CFG2)
    fake.info, fake.reason = [-1, -1, -1], [E.REASON_SINGULAR_PRECONDITIONER, E.REASON_INDEFINITE_MATRIX,
                                            E.REASON_SINGULAR_PRECONDITIONER]
    _, caught = _run(lambda: ml.solve_many(np.ones((N, 3)), accel="steepest_descent", maxiter=3))
    assert caught == [STOPS[1][2], STOPS[3][2]]
    fake.info = 0
    _, caught = _run(lambda: ml.solve_many(np.ones((N, 3)), accel="cgnr", maxiter=5000))
    assert caught == [CGN_CLAMP["cgnr"]]


@pytest.mark.parametrize("accel", ACCELS)
def test_batched_not_implemented_goes_column_by_column(load, fake, accel):
    ml = load(CFG9)
    n = 841
    entry = expected_call(accel, 3, n, 3)[0]
    fake.notimpl = {entry}
    fake.info, fake.reason = -1, E.REASON_INDEFINITE_MATRIX
    if accel == "steepest_descent":
        fake.reason = E.REASON_SINGULAR_PRECONDITIONER
    if accel in CGN_CLAMP:
        fake.info = 0                 # CGNR and CGNE have no info = -1 stop
    res = []
    (X, info), caught = _run(lambda: ml.solve_many(np.ones((n, 3)), tol=1e-7, maxiter=2000, cycle="W", accel=accel,
                                                   residuals=res, return_info=True))
    single = expected_call(accel, 2000, n)
    pre = [("amgb_hierarchy_set_transpose0", {}, None)] if accel in CGN_CLAMP else []
    batched = expected_call(accel, 2000, n, 3)
    assert fake.calls == pre + [batched] + [single] * 3
    assert np.array_equal(X, np.ones((n, 3))) and list(info) == [fake.info] * 3 and res == [[1.0, 0.5]] * 3
    want = []
    if accel == "cg":
        want = [SYM_WARNING, CG_STOP]
    elif accel == "bicgstab":
        want = [CG_STOP]
    elif accel in GMRES:
        want = [GMRES_CLAMP]
    elif accel in CGN_CLAMP:
        want = [CGN_CLAMP[accel]]
    if accel == "minimal_residual":
        want = [STOPS[0][2]]
    elif accel == "steepest_descent":
        want = [STOPS[3][2]]
    assert caught == want


@pytest.mark.parametrize("reorth", [False, True])
def test_krylov_gmres_mgs_reorth(load, fake, reorth):
    ml = load(CFG2)
    M = ml.aspreconditioner(cycle="W")
    x, info = krylov.gmres_mgs(ml.levels[0].A, np.ones((N, 1)), tol=1e-7, maxiter=4, M=M, reorth=reorth)
    flags = E.FLAG_X0_ZERO | E.FLAG_MGS | (E.FLAG_REORTH if reorth else 0)
    assert fake.calls == [("amgb_solve_gmres", dict(tol=1e-7, restart=0, maxiter=4, cycle=E.CYCLES["W"], flags=flags,
                                                     max_residuals=7), 7)]
    assert x.shape == (N, 1) and info == 0
    with pytest.raises(ValueError, match="AMLI cycles require acceleration"):
        krylov.gmres_mgs(ml.levels[0].A, np.ones(N), M=ml.aspreconditioner(cycle="AMLI"), reorth=True)
    one = load.one_by_one()
    with pytest.raises(NotImplementedError, match="reorth=True runs on real systems with n >= 2"):
        krylov.gmres_mgs(one.levels[0].A, np.ones(1), M=one.aspreconditioner(), reorth=True)
