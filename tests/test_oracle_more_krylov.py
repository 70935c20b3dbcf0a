"""oracle/krylov_more.py (CPU restatements of pyamg.krylov's CGNR, CGNE, minimal residual and steepest descent, driven by
the oracle's cycle as M) against what the real reference's ml.solve(accel=...) computed (tests/golden/krylov_more/,
written by make_golden_krylov_more.py): same iteration counts, info, residual histories and iterates on every
configuration."""
import os

import numpy as np
import pytest

import oracle
from oracle.krylov_more import run
from conftest import GOLDEN_ALL, GOLDEN_DIR, relerr

# tests/golden/make_golden_krylov_more.py RUNS
RUNS = {}
for _m, _c in (("cgnr", "W"), ("cgne", "F"), ("minimal_residual", "W"), ("steepest_descent", "F")):
    RUNS[_m] = dict(tol=1e-10, maxiter=8)
    RUNS[_m + "_x0"] = dict(tol=1e-3, maxiter=20, cycle=_c)
    RUNS[_m + "_zero"] = dict(tol=1e-8, maxiter=4)


def method_of(tag):
    return tag[:-3] if tag.endswith("_x0") else (tag[:-5] if tag.endswith("_zero") else tag)


def case(tag, ex):
    """(b, kw) of golden run `tag`: b = 0 for the *_zero runs, the stored x0 for the *_x0 runs."""
    kw = dict(RUNS[tag])
    b = ex["b"].ravel()
    if tag.endswith("_zero"):
        b = np.zeros_like(b)
    if tag.endswith("_x0"):
        kw["x0"] = ex["x0"].ravel()
    return b, kw


def check_against_golden(x, info, res, kg, tag):
    """iterate within relerr 1e-11 (NaN where the reference's is NaN), residual list within rtol 1e-7, equal info"""
    ref_x, ref_res = kg["x_ref_" + tag], kg["residuals_" + tag]
    assert info == int(kg["info_" + tag][0]), tag
    assert len(res) == len(ref_res), tag
    assert np.array_equal(np.isnan(res), np.isnan(ref_res)), tag
    ok = ~np.isnan(ref_res)
    assert np.allclose(np.asarray(res)[ok], ref_res[ok], rtol=1e-7, atol=1e-12 * ref_res[0]), tag
    if np.isnan(ref_x).any():
        assert np.isnan(x).all() and np.isnan(ref_x).all(), tag
    else:
        assert relerr(x, ref_x) < 1e-11, tag


@pytest.mark.parametrize("name", GOLDEN_ALL)
def test_oracle_more_krylov_matches_reference(name, load_golden):
    ml, ex = load_golden(name)
    kg = np.load(os.path.join(GOLDEN_DIR, "krylov_more", name + ".npz"))
    cyc = oracle.Cycle(oracle.hierarchy_spec(ml), coarse_pinv=ml.coarse_solver.P)
    for tag in RUNS:
        b, kw = case(tag, ex)
        res = []
        with np.errstate(invalid="ignore"):
            x, info = run(cyc, method_of(tag), b, residuals=res, **kw)
        check_against_golden(x, info, res, kg, tag)
