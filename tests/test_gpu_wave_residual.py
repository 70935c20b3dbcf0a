"""The residual after a Gauss-Seidel smoother, partly computed by the smoother's last wave (tile_kernels.cuh, OP_GS
with r): that wave's rows are final once it has run, so the launch that relaxes them also writes their residual
and the separate residual launch covers only the other waves.  Iterates must equal the separate residual launch
(AMGB_NO_WAVE_RESID=1) bit for bit; the stop test's norms are summed in another order and agree to rounding.

AMGB_TILE_MIN_NNZ=0 puts every wave on the tile kernel, so the small golden hierarchies take this path."""
import numpy as np
import pytest

from conftest import golden_path
from pyamg_b200.hierarchy_io import load_hierarchy

pytestmark = pytest.mark.gpu


def _solve(monkeypatch, name, fused, cycle="V", smoother=None, tol=0.0):
    monkeypatch.setenv("AMGB_TILE_MIN_NNZ", "0")
    if fused:
        monkeypatch.delenv("AMGB_NO_WAVE_RESID", raising=False)
    else:
        monkeypatch.setenv("AMGB_NO_WAVE_RESID", "1")
    ml, ex = load_hierarchy(golden_path(name))
    if smoother is not None:
        from pyamg_b200.relaxation.smoothing import change_smoothers
        change_smoothers(ml, smoother, smoother)
    res = []
    x = ml.solve(ex["b"], tol=tol, maxiter=3, cycle=cycle, residuals=res)
    x2 = ml.solve(ex["b"], tol=tol, maxiter=3, cycle=cycle)
    assert np.array_equal(x.view(np.int64), x2.view(np.int64))        # run to run
    ops = set(int(o) for o in ml.profile_cycle(cycle)[:, 1])
    return x, np.array(res), ops


def _same(monkeypatch, name, cycle="V", smoother=None, tol=0.0):
    xf, rf, of = _solve(monkeypatch, name, True, cycle, smoother, tol)
    xp, rp, op = _solve(monkeypatch, name, False, cycle, smoother, tol)
    assert 12 in of and 12 not in op, (of, op)
    assert np.array_equal(xf.view(np.int64), xp.view(np.int64))
    assert len(rf) == len(rp) and np.allclose(rf, rp, rtol=1e-14, atol=0)


@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg3_rs_mcgs_poisson3d", "cfg6_rs_gsfwd_none_poisson3d"])
@pytest.mark.parametrize("cycle", ["V", "W", "F"])
def test_last_wave_residual_bit_equal(monkeypatch, name, cycle):
    _same(monkeypatch, name, cycle)


@pytest.mark.parametrize("smoother", [("gauss_seidel", {"sweep": "forward", "iterations": 2}),
                                      ("gauss_seidel", {"sweep": "backward", "iterations": 2}),
                                      ("gauss_seidel", {"sweep": "symmetric", "iterations": 2}),
                                      ("sor", {"omega": 1.3, "sweep": "forward"}),
                                      ("sor", {"omega": 0.7, "sweep": "backward", "iterations": 2})])
def test_last_wave_residual_sweep_variants(monkeypatch, smoother):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", "V", smoother)


def test_last_wave_residual_stop_test(monkeypatch):
    _same(monkeypatch, "cfg3_rs_mcgs_poisson3d", "V", tol=1e-3)
