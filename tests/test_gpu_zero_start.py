"""The zero-start copy of a coarse level's operator (engine.cu build_zero_start): the first forward pass of a coarse
pre-smoother starts from x = +0, so wave w streams only each row's diagonal and its entries in earlier waves, kept
in the lanes and order of the full launch.  Iterates and residual lists must equal the full-operator launches
(AMGB_NO_ZERO_START=1) bit for bit.  The zero-start waves are profiled as op 13."""
import numpy as np
import pytest

from conftest import golden_path
from pyamg_b200.hierarchy_io import load_hierarchy

pytestmark = pytest.mark.gpu

ZERO_START_OP = 13


def _solve(monkeypatch, name, zero, cycle="V", smoother=None, tol=0.0, tiles_everywhere=False, x0=False,
           accel=None, edit=None):
    if tiles_everywhere:
        monkeypatch.setenv("AMGB_TILE_MIN_NNZ", "0")
    else:
        monkeypatch.delenv("AMGB_TILE_MIN_NNZ", raising=False)
    if zero:
        monkeypatch.delenv("AMGB_NO_ZERO_START", raising=False)
    else:
        monkeypatch.setenv("AMGB_NO_ZERO_START", "1")
    ml, ex = load_hierarchy(golden_path(name))
    if smoother is not None:
        from pyamg_b200.relaxation.smoothing import change_smoothers
        change_smoothers(ml, smoother, smoother)
    if edit is not None:
        edit(ml)
    res = []
    kw = dict(tol=tol, maxiter=3, cycle=cycle, residuals=res)
    if x0:
        kw["x0"] = ex["x0"].copy() if "x0" in ex else np.random.default_rng(7).random(ex["b"].size)
    if accel is not None:
        kw["accel"] = accel
    x = ml.solve(ex["b"], **kw)
    ops = set(int(o) for o in ml.profile_cycle(cycle)[:, 1])
    ml._invalidate()
    return x, np.array(res), ops


def _same(monkeypatch, name, expect=True, **kw):
    xz, rz, oz = _solve(monkeypatch, name, True, **kw)
    xf, rf, of = _solve(monkeypatch, name, False, **kw)
    assert ZERO_START_OP not in of, of
    assert (ZERO_START_OP in oz) == expect, oz
    assert np.array_equal(xz.view(np.int64), xf.view(np.int64))
    assert np.array_equal(rz.view(np.int64), rf.view(np.int64))


@pytest.mark.parametrize("tiles_everywhere", [False, True])
@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg3_rs_mcgs_poisson3d", "cfg6_rs_gsfwd_none_poisson3d"])
@pytest.mark.parametrize("cycle", ["V", "W", "F"])
def test_zero_start_bit_equal(monkeypatch, name, cycle, tiles_everywhere):
    _same(monkeypatch, name, cycle=cycle, tiles_everywhere=tiles_everywhere)


@pytest.mark.parametrize("smoother", [("gauss_seidel", {"sweep": "forward", "iterations": 2}),
                                      ("gauss_seidel", {"sweep": "symmetric", "iterations": 2}),
                                      ("sor", {"omega": 1.3, "sweep": "forward"}),
                                      ("sor", {"omega": 0.7, "sweep": "symmetric", "iterations": 2})])
@pytest.mark.parametrize("tiles_everywhere", [False, True])
def test_zero_start_sweep_variants(monkeypatch, smoother, tiles_everywhere):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", smoother=smoother, tiles_everywhere=tiles_everywhere)


def test_zero_start_backward_sweep_keeps_full_operator(monkeypatch):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", expect=False,
          smoother=("gauss_seidel", {"sweep": "backward", "iterations": 2}))


@pytest.mark.parametrize("tiles_everywhere", [False, True])
def test_zero_start_stop_test_and_x0(monkeypatch, tiles_everywhere):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", tol=1e-3, x0=True, tiles_everywhere=tiles_everywhere)


@pytest.mark.parametrize("accel", ["cg", "bicgstab"])
def test_zero_start_krylov(monkeypatch, accel):
    _same(monkeypatch, "cfg1_rs_gs_poisson2d", accel=accel, tol=1e-8)


def test_zero_start_zero_diagonal_row(monkeypatch):
    def edit(ml):
        A = ml.levels[1].A.tocsr(copy=True)
        A.data[np.flatnonzero(A.indices[A.indptr[3]:A.indptr[4]] == 3)[0] + A.indptr[3]] = 0.0
        ml.levels[1].A = A
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", edit=edit)


def test_zero_start_non_finite_entry_falls_back(monkeypatch):
    def edit(ml):
        for lvl in ml.levels[1:-1]:
            A = lvl.A.tocsr(copy=True)
            A.data[-1] = np.inf           # the last row's last entry: the cycle's values turn non-finite either way
            lvl.A = A
    xz, _, oz = _solve(monkeypatch, "cfg3_rs_mcgs_poisson3d", True, edit=edit)
    xf, _, of = _solve(monkeypatch, "cfg3_rs_mcgs_poisson3d", False, edit=edit)
    assert ZERO_START_OP not in oz and ZERO_START_OP not in of, (oz, of)
    assert np.array_equal(xz.view(np.int64), xf.view(np.int64))
