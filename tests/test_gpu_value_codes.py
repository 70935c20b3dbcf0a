"""Value codes (engine.cu upload_csr, tile_kernels.cuh CODED): a level operator with at most 256 distinct values (by
bit pattern) streams a one-byte code per entry into a table of those values on the tile kernels, instead of the
8-byte values.  Iterates and residual lists must equal the fp64 launches (AMGB_NO_VALUE_CODES=1) bit for bit.  The
profile charges a coded launch 5 B per entry plus the table instead of 12 B, which tells which launches ran coded."""
import numpy as np
import pytest

from conftest import golden_path
from pyamg_b200.hierarchy_io import load_hierarchy

pytestmark = pytest.mark.gpu

_KNOBS = ("AMGB_TILE_MIN_NNZ", "AMGB_TILE_FLAT", "AMGB_TILE_DENSE_CFG", "AMGB_NO_ZERO_START", "AMGB_NO_WAVE_RESID")


def _solve(monkeypatch, name, coded, cycle="V", smoother=None, tol=0.0, x0=False, accel=None, edit=None, env=None,
           many=False):
    env = dict(env or {})
    for k in _KNOBS:
        if k in env:
            monkeypatch.setenv(k, env[k])
        else:
            monkeypatch.delenv(k, raising=False)
    if coded:
        monkeypatch.delenv("AMGB_NO_VALUE_CODES", raising=False)
    else:
        monkeypatch.setenv("AMGB_NO_VALUE_CODES", "1")
    ml, ex = load_hierarchy(golden_path(name))
    if smoother is not None:
        from pyamg_b200.relaxation.smoothing import change_smoothers
        change_smoothers(ml, smoother, smoother)
    if edit is not None:
        edit(ml)
    b = ex["b"].ravel()
    if many:
        B = np.column_stack([b, np.random.default_rng(3).standard_normal(b.size), -2.0 * b])
        res = []
        x = ml.solve_many(B, tol=tol, maxiter=3, cycle=cycle, residuals=res, accel=accel)
        res = np.concatenate([np.asarray(r) for r in res])
    else:
        res = []
        kw = dict(tol=tol, maxiter=3, cycle=cycle, residuals=res)
        if x0:
            kw["x0"] = ex["x0"].copy() if "x0" in ex else np.random.default_rng(7).random(b.size)
        if accel is not None:
            kw["accel"] = accel
        x = ml.solve(b, **kw)
    prof = ml.profile_cycle(cycle)
    ml._invalidate()
    return x, np.asarray(res, dtype=np.float64), prof


def _same(monkeypatch, name, expect=True, **kw):
    """Bit-equal results both ways; returns the per-launch profile bytes (coded, fp64) and the launch records."""
    xc, rc, pc = _solve(monkeypatch, name, True, **kw)
    xf, rf, pf = _solve(monkeypatch, name, False, **kw)
    assert np.array_equal(xc.view(np.int64), xf.view(np.int64))
    assert np.array_equal(rc.view(np.int64), rf.view(np.int64))
    assert pc.shape == pf.shape and np.array_equal(pc[:, :4], pf[:, :4])     # the same launches, level, op, rows, nnz
    # a coded launch is charged 5 B per entry plus its table (1 to 256 doubles) instead of 12 B per entry
    coded = pc[:, 4] != pf[:, 4]
    table = 7.0 * pf[coded, 3] - (pf[coded, 4] - pc[coded, 4])
    assert ((table % 8 == 0) & (table >= 8) & (table <= 8 * 256)).all(), table
    assert (pc[coded, 4] < pf[coded, 4]).any() == expect, pc
    return pc, pf, coded


@pytest.mark.parametrize("tiles_everywhere", [False, True])
@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg3_rs_mcgs_poisson3d", "cfg6_rs_gsfwd_none_poisson3d"])
@pytest.mark.parametrize("cycle", ["V", "W", "F"])
def test_value_codes_gauss_seidel(monkeypatch, name, cycle, tiles_everywhere):
    env = {"AMGB_TILE_MIN_NNZ": "0"} if tiles_everywhere else {}
    _same(monkeypatch, name, expect=tiles_everywhere, cycle=cycle, env=env)


@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg4_sa_jacobi_aniso2d", "cfg7_sa_cheby_richardson_poisson2d",
                                  "cfg8_rs_cfjacobi_poisson3d", "cfg9_air_fcjacobi_advection2d"])
def test_value_codes_jacobi_polynomial_cf(monkeypatch, name):
    _same(monkeypatch, name, env={"AMGB_TILE_MIN_NNZ": "0"})


@pytest.mark.parametrize("flat", ["0", "1", "2"])
@pytest.mark.parametrize("dense", ["0", "7"])
@pytest.mark.parametrize("name", ["cfg3_rs_mcgs_poisson3d", "cfg2_sa_jacobi_poisson2d"])
def test_value_codes_kernel_variants(monkeypatch, name, flat, dense):
    _same(monkeypatch, name, env={"AMGB_TILE_MIN_NNZ": "0", "AMGB_TILE_FLAT": flat, "AMGB_TILE_DENSE_CFG": dense})


@pytest.mark.parametrize("no_zero_start", [False, True])
@pytest.mark.parametrize("no_wave_resid", [False, True])
def test_value_codes_zero_start_and_wave_residual(monkeypatch, no_zero_start, no_wave_resid):
    env = {"AMGB_TILE_MIN_NNZ": "0"}
    if no_zero_start:
        env["AMGB_NO_ZERO_START"] = "1"
    if no_wave_resid:
        env["AMGB_NO_WAVE_RESID"] = "1"
    pc, _, coded = _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", env=env)
    if not no_zero_start:
        assert coded[pc[:, 1] == 13].any(), pc          # a zero-start wave ran on the coded copy


@pytest.mark.parametrize("smoother", [("sor", {"omega": 1.3, "sweep": "forward"}),
                                      ("sor", {"omega": 0.7, "sweep": "symmetric", "iterations": 2})])
def test_value_codes_sor(monkeypatch, smoother):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", smoother=smoother, env={"AMGB_TILE_MIN_NNZ": "0"})


@pytest.mark.parametrize("tiles_everywhere", [False, True])
def test_value_codes_stop_test_and_x0(monkeypatch, tiles_everywhere):
    env = {"AMGB_TILE_MIN_NNZ": "0"} if tiles_everywhere else {}
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", expect=tiles_everywhere, tol=1e-3, x0=True, env=env)


@pytest.mark.parametrize("accel", ["cg", "bicgstab"])
def test_value_codes_krylov(monkeypatch, accel):
    _same(monkeypatch, "cfg1_rs_gs_poisson2d", accel=accel, tol=1e-8, env={"AMGB_TILE_MIN_NNZ": "0"})


@pytest.mark.parametrize("accel", [None, "cg"])
def test_value_codes_solve_many(monkeypatch, accel):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", many=True, accel=accel, env={"AMGB_TILE_MIN_NNZ": "0"})


def _distinct(a):
    return np.unique(np.ascontiguousarray(a).view(np.int64)).size


def _on_level0_A(pc):
    """Launches on level 0's A: residual, Jacobi and Gauss-Seidel waves (ops 0 and 2 are R and P)."""
    return (pc[:, 0] == 0) & np.isin(pc[:, 1], [1, 3, 4, 12, 13])


@pytest.mark.parametrize("ndistinct", [256, 257])
def test_value_codes_table_limit(monkeypatch, ndistinct):
    """A level with 256 distinct values is coded, one with 257 stays fp64."""
    def edit(ml):
        A = ml.levels[0].A.tocsr(copy=True)
        k = ndistinct - _distinct(A.data)
        # off-diagonal entries scaled by distinct factors: the original values stay present
        off = np.flatnonzero(A.indices != np.repeat(np.arange(A.shape[0]), np.diff(A.indptr)))[:k]
        A.data[off] *= 1.0 + (np.arange(k) + 1) * 2.0 ** -30
        assert _distinct(A.data) == ndistinct
        ml.levels[0].A = A
    pc, _, coded = _same(monkeypatch, "cfg1_rs_gs_poisson2d", edit=edit, env={"AMGB_TILE_MIN_NNZ": "0"})
    assert coded[_on_level0_A(pc)].any() == (ndistinct <= 256), pc


def test_value_codes_signed_zeros_and_non_finite(monkeypatch):
    """-0.0, +0.0, inf and NaN (with a payload) are distinct table entries and decode bit-exactly."""
    def edit(ml):
        A = ml.levels[0].A.tocsr(copy=True)
        off = np.flatnonzero(A.indices != np.repeat(np.arange(A.shape[0]), np.diff(A.indptr)))
        nan = np.array([0x7FF800000000BEEF], dtype=np.int64).view(np.float64)[0]
        A.data[off[-4:]] = [-0.0, 0.0, np.inf, nan]
        ml.levels[0].A = A
    pc, _, coded = _same(monkeypatch, "cfg1_rs_gs_poisson2d", edit=edit, env={"AMGB_TILE_MIN_NNZ": "0"})
    assert coded[_on_level0_A(pc)].any(), pc


def test_value_codes_mixed_levels(monkeypatch):
    """Levels whose operators all exceed 256 values stay fp64 while the others are coded, in one hierarchy."""
    name = "cfg3_rs_mcgs_poisson3d"
    ml, _ = load_hierarchy(golden_path(name))
    small = {l for l, lvl in enumerate(ml.levels[:-1])
             if min(_distinct(M.tocsr().data) for M in (lvl.A, lvl.P, lvl.R)) <= 256}
    ml._invalidate()
    assert small and len(small) < len(ml.levels) - 1, small
    pc, _, coded = _same(monkeypatch, name, env={"AMGB_TILE_MIN_NNZ": "0"})
    assert set(int(l) for l in pc[coded, 0]) == small, pc
