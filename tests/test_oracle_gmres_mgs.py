"""oracle/krylov_mgs.py (CPU restatement of pyamg.krylov.gmres_mgs, driven by the oracle's cycle as M) against what the
real reference computed (tests/golden/krylov_mgs/, written by make_golden_gmres_mgs.py): same iteration counts, info,
residual histories and iterates on every configuration."""
import os

import numpy as np
import pytest

import oracle
from oracle.krylov_mgs import run
from conftest import GOLDEN_ALL, GOLDEN_DIR, relerr

# tests/golden/make_golden_gmres_mgs.py RUNS
RUNS = {"mgs": dict(tol=1e-10, maxiter=12),
        "mgsW": dict(tol=1e-3, maxiter=25, cycle="W"),
        "mgsF": dict(tol=1e-4, maxiter=25, cycle="F"),
        "mgs_zero": dict(tol=1e-8, maxiter=6),
        "mgs_reorth": dict(tol=1e-10, maxiter=12),
        "mgs_stag": dict(tol=1e-30, maxiter=3)}


def case(tag, ex, kg):
    """(b, kw) of golden run `tag`, kw as ml.solve(accel='gmres_mgs') takes it (plus reorth for the reorth run)"""
    kw = dict(RUNS[tag])
    b = ex["b"].ravel()
    if tag in ("mgsW", "mgsF", "mgs_zero"):
        kw["x0"] = ex["x0"].ravel()
    if tag == "mgs_zero":
        b = np.zeros_like(b)
    if tag == "mgs_stag":
        b = kg["b_mgs_stag"]
        kw["x0"] = kg["x0_mgs_stag"]
    if tag == "mgs_reorth":
        kw["reorth"] = True
    return b, kw


def check_against_golden(x, info, res, kg, tag, x_bound=1e-11, res_rtol=1e-7):
    """equal info and residual count; iterate within x_bound (for b = 0 the iterate tends to zero: relative to
    the solution's scale, the W run's iterate); residual list within res_rtol, except for the stagnation run, whose residuals are rounding noise
    of b - A x (only the first is compared, loosely)"""
    ref_x, ref_res = kg["x_ref_" + tag], kg["residuals_" + tag]
    assert info == int(kg["info_" + tag][0]), tag
    assert len(res) == len(ref_res), tag
    if tag == "mgs_stag":
        assert np.allclose(res[0], ref_res[0], rtol=0.5), tag
        assert relerr(x, ref_x) < 1e-14, tag
        return
    assert np.allclose(res, ref_res, rtol=res_rtol, atol=1e-12 * ref_res[0]), tag
    if tag == "mgs_zero":
        assert np.linalg.norm(x - ref_x) < x_bound * np.linalg.norm(kg["x_ref_mgsW"]), tag
    else:
        assert relerr(x, ref_x) < x_bound, tag


@pytest.mark.parametrize("name", GOLDEN_ALL)
def test_oracle_gmres_mgs_matches_reference(name, load_golden):
    ml, ex = load_golden(name)
    kg = np.load(os.path.join(GOLDEN_DIR, "krylov_mgs", name + ".npz"))
    cyc = oracle.Cycle(oracle.hierarchy_spec(ml), coarse_pinv=ml.coarse_solver.P)
    for tag in RUNS:
        b, kw = case(tag, ex, kg)
        res = []
        x, info = run(cyc, b, residuals=res, **kw)
        check_against_golden(x, info, res, kg, tag)

