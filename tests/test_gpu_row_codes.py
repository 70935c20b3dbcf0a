"""Row codes (engine.cu upload_csr / row_codes, tile_kernels.cuh csr_rowcode_kernel): a pair-coded operator on one
lane per row whose rows take at most 256 distinct sequences of pair codes, none longer than 15 entries, streams one
byte per row naming its sequence.  Iterates and residual lists must equal the per-entry pair-code launches
(AMGB_NO_ROW_CODES=1) and the value-code launches (AMGB_NO_PAIR_CODES=1) bit for bit.  The profile charges a
row-coded launch 1 B per row plus its tile descriptors and tables, and no row pointers, which tells which launches
ran row-coded.  AMGB_ROW_MIN_NNZ=0 and AMGB_PAIR_MIN_NNZ=0 give row codes to the small test operators too."""
import numpy as np
import pytest

from conftest import golden_path
from pyamg_b200.hierarchy_io import load_hierarchy

pytestmark = pytest.mark.gpu

_KNOBS = ("AMGB_TILE_MIN_NNZ", "AMGB_NO_WAVE_RESID", "AMGB_ROW_MIN_NNZ", "AMGB_PAIR_MIN_NNZ")
_SMALL = {"AMGB_ROW_MIN_NNZ": "0", "AMGB_PAIR_MIN_NNZ": "0"}
_TILES = dict(_SMALL, AMGB_TILE_MIN_NNZ="0")


def _solve(monkeypatch, name, mode, cycle="V", tol=0.0, x0=False, accel=None, edit=None, env=None, many=False):
    env = dict(env or {})
    for k in _KNOBS:
        if k in env:
            monkeypatch.setenv(k, env[k])
        else:
            monkeypatch.delenv(k, raising=False)
    for k in ("AMGB_NO_VALUE_CODES", "AMGB_NO_PAIR_CODES", "AMGB_NO_ROW_CODES"):
        monkeypatch.delenv(k, raising=False)
    if mode == "pair":
        monkeypatch.setenv("AMGB_NO_ROW_CODES", "1")
    elif mode == "val8":
        monkeypatch.setenv("AMGB_NO_PAIR_CODES", "1")
    elif mode == "fp64":
        monkeypatch.setenv("AMGB_NO_VALUE_CODES", "1")
    ml, ex = load_hierarchy(golden_path(name))
    if edit is not None:
        edit(ml)
    b = ex["b"].ravel()
    res = []
    if many:
        B = np.column_stack([b, np.random.default_rng(3).standard_normal(b.size), -2.0 * b])
        x = ml.solve_many(B, tol=tol, maxiter=3, cycle=cycle, residuals=res, accel=accel)
        res = np.concatenate([np.asarray(r) for r in res])
    else:
        kw = dict(tol=tol, maxiter=3, cycle=cycle, residuals=res)
        if x0:
            kw["x0"] = np.random.default_rng(7).random(b.size)
        if accel is not None:
            kw["accel"] = accel
        x = ml.solve(b, **kw)
    prof = ml.profile_cycle(cycle)
    ml._invalidate()
    return x, np.asarray(res, dtype=np.float64), prof


def _on_level0_A(p):
    """Launches on level 0's A: residual, Jacobi and Gauss-Seidel waves (ops 0 and 2 are R and P)."""
    return (p[:, 0] == 0) & np.isin(p[:, 1], [1, 3, 4, 12, 13])


def _same(monkeypatch, name, expect=True, **kw):
    """Bit-equal results with row codes, per-entry pair codes and value codes; returns the row run's profile and
    which of its launches were row-coded."""
    xr, rr, pr = _solve(monkeypatch, name, "row", **kw)
    xp, rp, pp = _solve(monkeypatch, name, "pair", **kw)
    xv, rv, pv = _solve(monkeypatch, name, "val8", **kw)
    for x, r in ((xp, rp), (xv, rv)):
        assert np.array_equal(xr.view(np.int64), x.view(np.int64))
        assert np.array_equal(rr.view(np.int64), r.view(np.int64))
    assert pr.shape == pp.shape == pv.shape
    assert np.array_equal(pr[:, :4], pp[:, :4]) and np.array_equal(pr[:, :4], pv[:, :4])
    # a row-coded launch is charged 1 B per row, 8 B per tile descriptor (one more than the tiles) and 16 B per
    # pattern where the pair-coded one is charged 1 B per entry and a 4-B row pointer per row (plus one)
    rowed = pr[:, 4] != pp[:, 4]
    extra = pr[rowed, 4] - pp[rowed, 4] + pr[rowed, 3] + 3.0 * pr[rowed, 2]
    assert (((extra % 8 == 0) | (extra % 8 == 4)) & (extra >= 8 + 16)).all(), extra
    assert rowed.any() == expect, pr
    return pr, rowed


@pytest.mark.parametrize("tiles_everywhere", [False, True])
@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg3_rs_mcgs_poisson3d", "cfg6_rs_gsfwd_none_poisson3d"])
@pytest.mark.parametrize("cycle", ["V", "W", "F"])
def test_row_codes_gauss_seidel(monkeypatch, name, cycle, tiles_everywhere):
    """Gauss-Seidel waves, the last wave with its residual and the residual launches, under V, W and F cycles; with
    the default tile threshold the small goldens stay on the rows kernel and nothing is row-coded.  The forward
    sweep's wave order of cfg6 gives level 0 more than 256 distinct rows: it keeps per-entry pair codes."""
    rows_coded = tiles_everywhere and not name.startswith("cfg6")
    pr, rowed = _same(monkeypatch, name, expect=rows_coded, cycle=cycle, env=_TILES if tiles_everywhere else _SMALL)
    if rows_coded:
        assert rowed[_on_level0_A(pr)].all(), pr


@pytest.mark.parametrize("no_wave_resid", [False, True])
def test_row_codes_wave_residual(monkeypatch, no_wave_resid):
    env = dict(_TILES)
    if no_wave_resid:
        env["AMGB_NO_WAVE_RESID"] = "1"
    pr, rowed = _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", env=env)
    ops = set(int(o) for o in pr[rowed, 1])
    assert (12 in ops) != no_wave_resid, pr


def test_row_codes_stop_test_and_x0(monkeypatch):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", tol=1e-3, x0=True, env=_TILES)


@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg4_sa_jacobi_aniso2d"])
def test_row_codes_jacobi(monkeypatch, name):
    """Jacobi with and without its residual by-product, on the 5-point and the 9-point operator."""
    pr, rowed = _same(monkeypatch, name, env=_TILES)
    assert 3 in set(int(o) for o in pr[rowed, 1]), pr


@pytest.mark.parametrize("accel", ["cg", "bicgstab"])
def test_row_codes_krylov(monkeypatch, accel):
    _same(monkeypatch, "cfg1_rs_gs_poisson2d", accel=accel, tol=1e-8, env=_TILES)


def test_row_codes_solve_many(monkeypatch):
    """solve_many streams Aj / Ax itself: its results do not depend on the codes."""
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", many=True, env=_TILES)


def _rows(A):
    return np.repeat(np.arange(A.shape[0]), np.diff(A.indptr))


def _patterns(A):
    """Distinct rows as sequences of (value bits, column - row) in stored order."""
    d = A.indices.astype(np.int64) - _rows(A)
    v = A.data.view(np.int64)
    return len({(tuple(v[s:e]), tuple(d[s:e])) for s, e in zip(A.indptr[:-1], A.indptr[1:])})


def _pairs(A):
    return len(set(zip(A.data.view(np.int64), A.indices.astype(np.int64) - _rows(A))))


def _offdiag(A):
    return np.flatnonzero(A.indices != _rows(A))


@pytest.mark.parametrize("npat", [256, 257])
def test_row_codes_pattern_limit(monkeypatch, npat):
    """256 row patterns are row-coded; 257 (with at most 256 pairs) fall back to per-entry pair codes.  Each new
    pattern is an interior row with one entry given a value of its own.  Level 0 of the Jacobi hierarchy keeps its
    natural row order, so the patterns counted here are the uploaded ones."""
    def edit(ml):
        A = ml.levels[0].A.tocsr(copy=True)
        k = npat - _patterns(A)
        interior = np.flatnonzero(np.diff(A.indptr) == 5)
        rows = interior[len(interior) // 2 - k // 2:][:k]
        A.data[A.indptr[rows]] *= 1.0 + (np.arange(k) + 1) * 2.0 ** -30
        assert _patterns(A) == npat and _pairs(A) <= 256
        ml.levels[0].A = A
    _same(monkeypatch, "cfg2_sa_jacobi_poisson2d", expect=npat <= 256, edit=edit, env=_TILES)


@pytest.mark.parametrize("length", [15, 16])
def test_row_codes_row_length_cap(monkeypatch, length):
    """A row of 15 entries is row-coded; one of 16 leaves the operator on per-entry pair codes."""
    import scipy.sparse as sp

    def edit(ml):
        A = ml.levels[0].A.tocsr(copy=True).tolil()
        n = A.shape[0]
        i = n // 2
        cols = [c for c in range(i - 40, i + 40) if c != i and A[i, c] == 0][:length - A[i].nnz]
        for c in cols:
            A[i, c] = -1e-3
        A = sp.csr_matrix(A)
        assert np.diff(A.indptr).max() == length
        ml.levels[0].A = A
    _same(monkeypatch, "cfg2_sa_jacobi_poisson2d", expect=length <= 15, edit=edit, env=_TILES)


@pytest.mark.parametrize("case", ["duplicate_diagonal", "zero_diagonal", "missing_diagonal", "signed_zeros_nan"])
def test_row_codes_special_entries(monkeypatch, case):
    """A duplicated diagonal entry (the last one wins), a zero diagonal and a missing one (the row keeps its x), and
    -0.0 / +0.0 / NaN with a payload as distinct pairs that decode bit-exactly."""
    import scipy.sparse as sp

    def edit(ml):
        A = ml.levels[0].A.tocsr(copy=True)
        n = A.shape[0]
        if case == "duplicate_diagonal":
            rows = _rows(A)
            extra = np.arange(0, n, 7)
            r = np.concatenate([rows, extra])
            c = np.concatenate([A.indices, extra])
            v = np.concatenate([A.data, np.full(extra.size, 3.0)])
            o = np.lexsort((np.arange(r.size), r))
            A = sp.csr_matrix((v[o], c[o], np.r_[0, np.cumsum(np.bincount(r, minlength=n))]), shape=A.shape)
            A.has_sorted_indices = False
        elif case == "zero_diagonal":
            d = np.flatnonzero(A.indices == _rows(A))
            A.data[d[::5]] = 0.0
        elif case == "missing_diagonal":
            d = np.flatnonzero(A.indices == _rows(A))
            keep = np.ones(A.nnz, dtype=bool)
            keep[d[::9]] = False
            r = _rows(A)[keep]
            A = sp.csr_matrix((A.data[keep], A.indices[keep], np.r_[0, np.cumsum(np.bincount(r, minlength=n))]),
                              shape=A.shape)
        else:
            nan = np.array([0x7FF800000000BEEF], dtype=np.int64).view(np.float64)[0]
            A.data[_offdiag(A)[-3:]] = [-0.0, 0.0, nan]
        ml.levels[0].A = A
    _same(monkeypatch, "cfg2_sa_jacobi_poisson2d", edit=edit, env=_TILES)


def test_row_codes_mixed_kinds(monkeypatch):
    """One hierarchy with row-coded, value-coded and fp64 operators: row codes on level 0's A but not on level 1 (its
    rows are irregular; a coarse level small enough to have few patterns may qualify)."""
    name = "cfg3_rs_mcgs_poisson3d"
    pr, rowed = _same(monkeypatch, name, env=_TILES)
    _, _, pp = _solve(monkeypatch, name, "pair", env=_TILES)
    _, _, pv = _solve(monkeypatch, name, "val8", env=_TILES)
    _, _, pf = _solve(monkeypatch, name, "fp64", env=_TILES)
    paired = (pp[:, 4] != pv[:, 4]) & ~rowed
    valued = (pv[:, 4] != pf[:, 4]) & ~rowed & ~paired
    levels = set(int(l) for l in pr[rowed, 0])
    assert 0 in levels and 1 not in levels, pr
    assert valued.any() and (~rowed & ~paired & ~valued).any(), pr


def test_row_codes_default_threshold(monkeypatch):
    """Without AMGB_ROW_MIN_NNZ, operators below the default tile threshold keep per-entry pair codes."""
    env = dict(_TILES)
    del env["AMGB_ROW_MIN_NNZ"]
    _, _, pr = _solve(monkeypatch, "cfg3_rs_mcgs_poisson3d", "row", env=env)
    _, _, pp = _solve(monkeypatch, "cfg3_rs_mcgs_poisson3d", "pair", env=env)
    assert np.array_equal(pr[:, :5], pp[:, :5])
