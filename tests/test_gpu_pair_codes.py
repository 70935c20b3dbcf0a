"""Pair codes (engine.cu upload_csr / pair_codes, tile_kernels.cuh CODE_PAIR8): an operator on the lanes-per-row tile
kernel whose entries take at most 256 distinct (value bit pattern, column - row) pairs streams one byte per entry
into a table of those pairs, instead of a value code and a 4-byte column.  Iterates and residual lists must equal
both the value-code launches (AMGB_NO_PAIR_CODES=1) and the fp64 launches (AMGB_NO_VALUE_CODES=1) bit for bit.  The
profile charges a pair-coded launch 1 B per entry plus 16 B per pair, which tells which launches ran pair-coded.
AMGB_PAIR_MIN_NNZ=0 gives pair codes to the small test operators too."""
import numpy as np
import pytest

from conftest import golden_path
from pyamg_b200.hierarchy_io import load_hierarchy

pytestmark = pytest.mark.gpu

_KNOBS = ("AMGB_TILE_MIN_NNZ", "AMGB_TILE_FLAT", "AMGB_TILE_DENSE_CFG", "AMGB_NO_ZERO_START", "AMGB_NO_WAVE_RESID",
          "AMGB_TILE_G")
_TILES = {"AMGB_TILE_MIN_NNZ": "0"}


def _solve(monkeypatch, name, mode, cycle="V", tol=0.0, x0=False, accel=None, edit=None, env=None, many=False):
    env = dict(env or {})
    for k in _KNOBS:
        if k in env:
            monkeypatch.setenv(k, env[k])
        else:
            monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("AMGB_PAIR_MIN_NNZ", "0")
    monkeypatch.delenv("AMGB_NO_VALUE_CODES", raising=False)
    monkeypatch.delenv("AMGB_NO_PAIR_CODES", raising=False)
    if mode == "val8":
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


def _same(monkeypatch, name, expect=True, **kw):
    """Bit-equal results in all three modes; returns the pair run's profile and which of its launches were
    pair-coded."""
    xp, rp, pp = _solve(monkeypatch, name, "pair", **kw)
    xv, rv, pv = _solve(monkeypatch, name, "val8", **kw)
    xf, rf, pf = _solve(monkeypatch, name, "fp64", **kw)
    for x, r in ((xv, rv), (xf, rf)):
        assert np.array_equal(xp.view(np.int64), x.view(np.int64))
        assert np.array_equal(rp.view(np.int64), r.view(np.int64))
    assert pp.shape == pv.shape == pf.shape
    assert np.array_equal(pp[:, :4], pf[:, :4]) and np.array_equal(pv[:, :4], pf[:, :4])
    # a pair-coded launch is charged 1 B per entry plus 16 B per pair (1 to 256) instead of 12 B per entry
    paired = pp[:, 4] != pv[:, 4]
    table = pp[paired, 4] - pf[paired, 4] + 11.0 * pf[paired, 3]
    assert ((table % 16 == 0) & (table >= 16) & (table <= 16 * 256)).all(), table
    assert paired.any() == expect, pp
    return pp, paired


def _on_level0_A(p):
    """Launches on level 0's A: residual, Jacobi and Gauss-Seidel waves (ops 0 and 2 are R and P)."""
    return (p[:, 0] == 0) & np.isin(p[:, 1], [1, 3, 4, 12, 13])


@pytest.mark.parametrize("tiles_everywhere", [False, True])
@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg3_rs_mcgs_poisson3d", "cfg6_rs_gsfwd_none_poisson3d"])
@pytest.mark.parametrize("cycle", ["V", "W", "F"])
def test_pair_codes_gauss_seidel(monkeypatch, name, cycle, tiles_everywhere):
    """Gauss-Seidel waves, the last wave with its residual, residual / restriction / prolongation launches."""
    pp, paired = _same(monkeypatch, name, expect=tiles_everywhere, cycle=cycle,
                       env=_TILES if tiles_everywhere else {})
    if tiles_everywhere:
        assert paired[_on_level0_A(pp)].all(), pp


@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg4_sa_jacobi_aniso2d", "cfg7_sa_cheby_richardson_poisson2d",
                                  "cfg8_rs_cfjacobi_poisson3d"])
def test_pair_codes_jacobi_polynomial_cf(monkeypatch, name):
    """Jacobi with and without its residual by-product, SpMV of the polynomial smoother, C/F Jacobi."""
    _same(monkeypatch, name, env=_TILES)


@pytest.mark.parametrize("flat", ["0", "2"])
@pytest.mark.parametrize("dense", ["0", "7"])
def test_pair_codes_kernel_variants(monkeypatch, flat, dense):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", env=dict(_TILES, AMGB_TILE_FLAT=flat, AMGB_TILE_DENSE_CFG=dense))


@pytest.mark.parametrize("G", ["2", "4"])
def test_pair_codes_lanes_per_row(monkeypatch, G):
    """More than one lane per row: the group sum and the diagonal search across lanes."""
    pp, paired = _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", env=dict(_TILES, AMGB_TILE_G=G))
    assert paired[_on_level0_A(pp)].all(), pp


@pytest.mark.parametrize("no_wave_resid", [False, True])
def test_pair_codes_zero_start_and_wave_residual(monkeypatch, no_wave_resid):
    env = dict(_TILES)
    if no_wave_resid:
        env["AMGB_NO_WAVE_RESID"] = "1"
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", env=env)


def test_pair_codes_stop_test_and_x0(monkeypatch):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", tol=1e-3, x0=True, env=_TILES)


@pytest.mark.parametrize("accel", ["cg", "bicgstab"])
def test_pair_codes_krylov(monkeypatch, accel):
    _same(monkeypatch, "cfg1_rs_gs_poisson2d", accel=accel, tol=1e-8, env=_TILES)


def test_pair_codes_solve_many(monkeypatch):
    """solve_many streams Aj / Ax itself: its results do not depend on the codes."""
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", many=True, env=_TILES)


def _offdiag(A):
    return np.flatnonzero(A.indices != np.repeat(np.arange(A.shape[0]), np.diff(A.indptr)))


def _pairs(A):
    rows = np.repeat(np.arange(A.shape[0]), np.diff(A.indptr))
    key = np.stack([A.data.view(np.int64), A.indices.astype(np.int64) - rows])
    return np.unique(key, axis=1).shape[1]


@pytest.mark.parametrize("npairs", [256, 257])
def test_pair_codes_table_limit(monkeypatch, npairs):
    """256 pairs are pair-coded; 257 (with at most 256 values) fall back to value codes.  Level 0 of the Jacobi
    hierarchy keeps its natural row order, so the pairs counted here are the uploaded ones."""
    def edit(ml):
        A = ml.levels[0].A.tocsr(copy=True)
        k = npairs - _pairs(A)
        off = _offdiag(A)[:k]           # each a new value, so each a new pair
        A.data[off] *= 1.0 + (np.arange(k) + 1) * 2.0 ** -30
        assert _pairs(A) == npairs and np.unique(A.data.view(np.int64)).size <= 256
        ml.levels[0].A = A
    pp, paired = _same(monkeypatch, "cfg2_sa_jacobi_poisson2d", expect=npairs <= 256, edit=edit, env=_TILES)
    assert paired[_on_level0_A(pp)].any() == (npairs <= 256), pp


@pytest.mark.parametrize("case", ["duplicate_diagonal", "zero_diagonal", "signed_zeros_nan"])
def test_pair_codes_special_entries(monkeypatch, case):
    """A duplicated diagonal entry (the last one wins), a zero diagonal (the row keeps its x), and -0.0 / +0.0 /
    NaN with a payload as distinct pairs that decode bit-exactly."""
    import scipy.sparse as sp

    def edit(ml):
        A = ml.levels[0].A.tocsr(copy=True)
        if case == "duplicate_diagonal":
            n = A.shape[0]
            rows = np.repeat(np.arange(n), np.diff(A.indptr))
            extra = np.arange(0, n, 7)
            r = np.concatenate([rows, extra])
            c = np.concatenate([A.indices, extra])
            v = np.concatenate([A.data, np.full(extra.size, 3.0)])
            o = np.lexsort((np.arange(r.size), r))
            A = sp.csr_matrix((v[o], c[o], np.r_[0, np.cumsum(np.bincount(r, minlength=n))]), shape=A.shape)
            A.has_sorted_indices = False
        elif case == "zero_diagonal":
            d = np.flatnonzero(A.indices == np.repeat(np.arange(A.shape[0]), np.diff(A.indptr)))
            A.data[d[::5]] = 0.0
        else:
            nan = np.array([0x7FF800000000BEEF], dtype=np.int64).view(np.float64)[0]
            A.data[_offdiag(A)[-3:]] = [-0.0, 0.0, nan]
        ml.levels[0].A = A
    pp, paired = _same(monkeypatch, "cfg2_sa_jacobi_poisson2d", edit=edit, env=_TILES)
    assert paired[_on_level0_A(pp)].any(), pp


def test_pair_codes_long_rows(monkeypatch):
    """Rows longer than a tile (224 entries) stream their codes from global memory."""
    import scipy.sparse as sp

    def edit(ml):
        A = ml.levels[0].A.tocsr(copy=True).tolil()
        n = A.shape[0]
        i = n // 2              # one row of 240 entries: each a new column offset, and still at most 256 pairs
        cols = np.linspace(0, n - 1, 240).astype(int)
        A[i, cols[cols != i]] = -1e-3
        ml.levels[0].A = sp.csr_matrix(A)
    pp, paired = _same(monkeypatch, "cfg2_sa_jacobi_poisson2d", edit=edit, env=_TILES)
    assert paired[_on_level0_A(pp)].any(), pp


def test_pair_codes_mixed_kinds(monkeypatch):
    """One hierarchy with pair-coded, value-coded and fp64 operators: pair codes on level 0's A but not on level 1
    (its column offsets are irregular; a coarse level small enough to have few entries may qualify), value codes
    where an operator has at most 256 values."""
    name = "cfg3_rs_mcgs_poisson3d"
    pp, paired = _same(monkeypatch, name, env=_TILES)
    _, _, pv = _solve(monkeypatch, name, "val8", env=_TILES)
    _, _, pf = _solve(monkeypatch, name, "fp64", env=_TILES)
    valued = (pv[:, 4] != pf[:, 4]) & ~paired
    levels = set(int(l) for l in pp[paired, 0])
    assert 0 in levels and 1 not in levels, pp
    assert valued.any() and (~paired & ~valued).any(), pp


def test_pair_codes_default_threshold(monkeypatch):
    """Without AMGB_PAIR_MIN_NNZ, operators below the default tile threshold keep value codes."""
    monkeypatch.setenv("AMGB_TILE_MIN_NNZ", "0")
    monkeypatch.delenv("AMGB_NO_PAIR_CODES", raising=False)
    monkeypatch.delenv("AMGB_NO_VALUE_CODES", raising=False)
    monkeypatch.delenv("AMGB_PAIR_MIN_NNZ", raising=False)
    ml, ex = load_hierarchy(golden_path("cfg3_rs_mcgs_poisson3d"))
    ml.solve(ex["b"].ravel(), tol=0.0, maxiter=1)
    p = ml.profile_cycle("V")
    ml._invalidate()
    A0 = _on_level0_A(p)
    assert (p[A0, 4] > 4.0 * p[A0, 3]).all(), p          # at least 5 B per entry: not pair-coded
