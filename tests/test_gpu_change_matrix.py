"""MultilevelSolver.change_solve_matrix on a resident hierarchy (amgb_hierarchy_replace_level0): only level 0 is
replaced on the device -- values refreshed in place for a same-pattern change (path 1), level 0 rebuilt otherwise
(path 2) -- and every later solve returns, bit for bit, what a hierarchy uploaded from scratch on the same levels
returns: iterates, info and residual lists of solve (V / W / F / AMLI), solve_many and the resident Krylov methods."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import GOLDEN_ALL, golden_path
from pyamg_b200.hierarchy_io import load_hierarchy
from pyamg_b200.multilevel import MultilevelSolver

pytestmark = pytest.mark.gpu

MULTILEVEL = [g for g in GOLDEN_ALL if len(load_hierarchy(golden_path(g))[0].levels) >= 2]


def _load(name):
    """A golden hierarchy; level 0 gets the CF splitting its stored CF / FC Jacobi smoothers were set up with (the
    stored levels do not carry it, and rebuild_smoother needs it, as in the reference)."""
    ml, ex = load_hierarchy(golden_path(name))
    for sm in (ml.levels[0].presmoother, ml.levels[0].postsmoother):
        kw = getattr(sm, "keywords", {})
        if "Cpts" in kw and not hasattr(ml.levels[0], "splitting"):
            splitting = np.zeros(ml.levels[0].A.shape[0], dtype=bool)
            splitting[kw["Cpts"]] = True
            ml.levels[0].splitting = splitting
    return ml, ex


def _fresh(ml):
    """A new solver on the same levels (level 0 = the changed matrix and its rebuilt smoothers), uploaded from scratch."""
    return MultilevelSolver.from_pyamg(ml)


def _bits(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.float64)).view(np.int64)


def _outputs(ml, b, cycles=("V", "W", "F", "AMLI"), accels=("cg", "gmres", "fgmres", "cgnr"), ks=(3, 8)):
    """Everything the solve paths return on b; a path the hierarchy does not support records its exception type."""
    out = {}

    def run(key, fn):
        try:
            out[key] = fn()
        except NotImplementedError as exc:
            out[key] = type(exc).__name__

    def single(**kw):
        res = []
        x, info = ml.solve(b, tol=1e-10, maxiter=4, residuals=res, return_info=True, **kw)
        return _bits(x), info, _bits(res)

    def many(k, **kw):
        B = np.column_stack([b * (j + 1) + j for j in range(k)])
        res = []
        X, info = ml.solve_many(B, tol=1e-10, maxiter=4, residuals=res, return_info=True, **kw)
        return _bits(X), np.asarray(info).tolist(), [_bits(r) for r in res]

    for c in cycles:
        run(("solve", c), lambda c=c: single(cycle=c))
    for a in accels:
        run(("accel", a), lambda a=a: single(accel=a))
    for k in ks:
        run(("many", k), lambda k=k: many(k))
    run(("many-cg", 3), lambda: many(3, accel="cg"))
    return out


def _same(a, b):
    assert a.keys() == b.keys()
    for key in a:
        x, y = a[key], b[key]
        if isinstance(x, str) or isinstance(y, str):
            assert x == y, key
            continue
        assert np.array_equal(x[0], y[0]), key
        assert x[1] == y[1], key
        if isinstance(x[2], list):
            assert len(x[2]) == len(y[2]) and all(np.array_equal(p, q) for p, q in zip(x[2], y[2])), key
        else:
            assert np.array_equal(x[2], y[2]), key


def _settle(ml):
    """change_solve_matrix to the matrix level 0 already has: rebuild_smoother sets the smoothers up from their names
    with default options (as the reference does), which may differ from the ones the hierarchy was built with, so
    that first change may rebuild level 0; after it the smoothers' structure is the one later changes keep."""
    ml.upload()
    ml.change_solve_matrix(ml.levels[0].A)


def _check_change(ml, b, A2, expect_path=None, **kw):
    ml.upload()
    ml.change_solve_matrix(A2)
    path = ml._last_replace_path
    if expect_path is not None:
        assert path == expect_path
    got = _outputs(ml, b, **kw)
    want = _outputs(_fresh(ml), b, **kw)
    _same(got, want)
    return path


def _shifted(A, seed=0):
    """A + diag(d), distinct positive d: the pattern of A (with its diagonal), more distinct values."""
    A = sp.csr_matrix(A)
    d = 1.0 + np.random.default_rng(seed).permutation(A.shape[0]) / A.shape[0]
    B = (A + sp.diags(d)).tocsr()
    return B if B.nnz == A.nnz else None


@pytest.mark.parametrize("name", MULTILEVEL)
def test_scaled_matrix_refreshes_in_place(name):
    ml, ex = _load(name)
    _settle(ml)
    _check_change(ml, ex["b"], 2.0 * ml.levels[0].A, expect_path=1)


@pytest.mark.parametrize("name", MULTILEVEL)
def test_shifted_matrix(name):
    ml, ex = _load(name)
    A2 = _shifted(ml.levels[0].A)
    if A2 is None:
        pytest.skip("level 0 has no stored diagonal")
    assert _check_change(ml, ex["b"], A2) in (1, 2)


def _pattern_change(A, drop):
    """A with one symmetric off-diagonal pair dropped (its weight moved onto the diagonal: still SPD) or added."""
    A = sp.csr_matrix(A).tolil()
    n = A.shape[0]
    if drop:
        C = sp.triu(sp.csr_matrix(A), k=1).tocoo()
        i, j, v = int(C.row[0]), int(C.col[0]), float(C.data[0])
        A[i, j] = 0.0
        A[j, i] = 0.0
        A[i, i] += abs(v)
        A[j, j] += abs(v)
        B = sp.csr_matrix(A)
        B.eliminate_zeros()
        return B
    i, j = 0, n - 1
    A[i, j] = -1e-3
    A[j, i] = -1e-3
    A[i, i] += 1e-3
    A[j, j] += 1e-3
    return sp.csr_matrix(A)


@pytest.mark.parametrize("drop", [True, False])
@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg2_sa_jacobi_poisson2d", "cfg3_rs_mcgs_poisson3d"])
def test_pattern_change_rebuilds_level0(name, drop):
    ml, ex = _load(name)
    _check_change(ml, ex["b"], _pattern_change(ml.levels[0].A, drop), expect_path=2)


def test_alternating_changes():
    ml, ex = _load("cfg3_rs_mcgs_poisson3d")
    b = ex["b"]
    _settle(ml)
    A1 = sp.csr_matrix(ml.levels[0].A)
    mats = [1.5 * A1, _pattern_change(A1, False)]
    want = []
    for A in mats:
        ml.change_solve_matrix(A)
        want.append(_outputs(_fresh(ml), b, cycles=("V", "W"), accels=("cg",), ks=(3,)))
    for step in range(10):
        ml.change_solve_matrix(mats[step % 2])
        assert ml._last_replace_path == 2
        _same(_outputs(ml, b, cycles=("V", "W"), accels=("cg",), ks=(3,)), want[step % 2])
    ml.change_solve_matrix(A1)
    for step in range(4):                               # same pattern, alternating values: in place every time
        ml.change_solve_matrix((2.0 - step % 2) * A1)
        assert ml._last_replace_path == 1
        got = _outputs(ml, b, cycles=("V",), accels=("cg",), ks=(3,))
        _same(got, _outputs(_fresh(ml), b, cycles=("V",), accels=("cg",), ks=(3,)))


def test_changed_hierarchy_matches_oracle():
    import oracle
    ml, ex = _load("cfg3_rs_mcgs_poisson3d")
    ml.upload()
    ml.change_solve_matrix(_shifted(ml.levels[0].A))
    x = ml.solve(ex["b"], tol=0, maxiter=3)
    cyc = oracle.Cycle(oracle.hierarchy_spec(ml), coarse_pinv=ml.coarse_solver.P)
    xo = cyc.solve(ex["b"], tol=0, maxiter=3)
    assert np.linalg.norm(x - xo) / np.linalg.norm(xo) < 1e-12


FORMATS = [
    {},
    {"AMGB_TILE_MIN_NNZ": "0"},
    {"AMGB_TILE_MIN_NNZ": "0", "AMGB_PAIR_MIN_NNZ": "0"},
    {"AMGB_TILE_MIN_NNZ": "0", "AMGB_PAIR_MIN_NNZ": "0", "AMGB_ROW_MIN_NNZ": "0"},
    {"AMGB_TILE_MIN_NNZ": "0", "AMGB_PAIR_MIN_NNZ": "0", "AMGB_ROW_MIN_NNZ": "0", "AMGB_NO_ROW_CODES": "1"},
    {"AMGB_TILE_MIN_NNZ": "0", "AMGB_NO_PAIR_CODES": "1"},
    {"AMGB_TILE_MIN_NNZ": "0", "AMGB_NO_PAIR_CODES": "1", "AMGB_NO_VALUE_CODES": "1"},
    {"AMGB_NO_TILES": "1"},
    {"AMGB_NO_PERMUTE": "1", "AMGB_TILE_MIN_NNZ": "0"},
    {"AMGB_NO_GRAPH": "1", "AMGB_TILE_MIN_NNZ": "0", "AMGB_PAIR_MIN_NNZ": "0", "AMGB_ROW_MIN_NNZ": "0"},
]


@pytest.mark.parametrize("env", FORMATS, ids=lambda e: ",".join(f"{k[5:]}={v}" for k, v in e.items()) or "default")
@pytest.mark.parametrize("name", ["cfg3_rs_mcgs_poisson3d", "cfg2_sa_jacobi_poisson2d"])
def test_every_level0_stream_format(monkeypatch, name, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ml, ex = _load(name)
    _settle(ml)
    A = ml.levels[0].A
    _check_change(ml, ex["b"], 2.0 * A, expect_path=1, cycles=("V", "W"), accels=("cg",), ks=(3,))
    path = _check_change(ml, ex["b"], _shifted(A, 1), cycles=("V", "W"), accels=("cg",), ks=(3,))
    if env.get("AMGB_NO_VALUE_CODES") == "1" or env.get("AMGB_NO_TILES") == "1":
        assert path == 1                                # fp64 values stay fp64
    _check_change(ml, ex["b"], _pattern_change(A, True), expect_path=2, cycles=("V",), accels=("cg",), ks=(3,))


SMOOTHERS = [
    ("cfg2_sa_jacobi_poisson2d", ("jacobi", {"withrho": True, "omega": 4.0 / 3.0})),
    ("cfg1_rs_gs_poisson2d", ("gauss_seidel", {"sweep": "symmetric"})),
    ("cfg3_rs_mcgs_poisson3d", None),                   # multi-colour Gauss-Seidel: row lists
    ("cfg5_sa_bjacobi_elasticity", None),               # block Jacobi
    ("cfg10_sa_bgs_elasticity", None),                  # block Gauss-Seidel
    ("cfg7_sa_cheby_richardson_poisson2d", None),       # Chebyshev / Richardson
    ("cfg8_rs_cfjacobi_poisson3d", None),               # CF Jacobi
    ("cfg9_air_fcjacobi_advection2d", None),            # FC Jacobi
    ("cfg12_sa_sor_poisson2d", None),
    ("cfg13_rs_gsnr_gsne_advdiff2d", None),             # Gauss-Seidel NR / NE
    ("cfg14_sa_jacobine_poisson2d", None),              # Jacobi NE
    ("cfg15_sa_schwarz_aniso2d", None),                 # Schwarz
]


@pytest.mark.parametrize("name,smoother", SMOOTHERS, ids=[s[0] for s in SMOOTHERS])
def test_every_level0_smoother_kind(name, smoother):
    ml, ex = _load(name)
    if smoother is not None:
        from pyamg_b200.relaxation.smoothing import change_smoothers
        change_smoothers(ml, smoother, smoother)
    _settle(ml)
    A = ml.levels[0].A
    _check_change(ml, ex["b"], 3.0 * A, expect_path=1, ks=(3,))
    A2 = _shifted(A, 2)
    if A2 is not None:
        _check_change(ml, ex["b"], A2, ks=(3,))


def test_cuda_tensors_after_change():
    torch = pytest.importorskip("torch")
    ml, ex = _load("cfg3_rs_mcgs_poisson3d")
    _settle(ml)
    ml.change_solve_matrix(2.0 * ml.levels[0].A)
    assert ml._last_replace_path == 1
    fresh = _fresh(ml)
    b = torch.tensor(ex["b"], dtype=torch.float64, device="cuda")
    for accel in (None, "cg", "gmres"):
        r1, r2 = [], []
        x1 = ml.solve(b, tol=1e-10, maxiter=4, accel=accel, residuals=r1)
        x2 = fresh.solve(b, tol=1e-10, maxiter=4, accel=accel, residuals=r2)
        assert torch.equal(x1, x2) and r1 == r2, accel


def test_one_level_hierarchy_falls_back():
    from pyamg_b200.classical import ruge_stuben_solver
    from pyamg_b200.gallery import poisson
    A = poisson((6, 6), format="csr")
    ml = ruge_stuben_solver(A, max_coarse=1000)
    assert len(ml.levels) == 1
    from pyamg_b200.relaxation.smoothing import setup_gauss_seidel
    ml.levels[0].presmoother = setup_gauss_seidel(ml.levels[0])
    ml.levels[0].postsmoother = setup_gauss_seidel(ml.levels[0])
    b = np.arange(A.shape[0], dtype=float)
    ml.solve(b, maxiter=2)
    ml.change_solve_matrix(2.0 * A)
    assert ml._last_replace_path == 0
    _same(_outputs(ml, b, accels=("cg",), ks=(3,)), _outputs(_fresh(ml), b, accels=("cg",), ks=(3,)))
