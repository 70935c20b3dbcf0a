"""Generate tests/golden/krylov_more/<cfg>.npz by running the REAL reference (see make_golden.py):

    AMGB_REFERENCE=<reference checkout> python oracle/build.py
    PYTHONPATH=oracle/_ref/site python tests/golden/make_golden_krylov_more.py

Rebuilds make_golden.py's hierarchies exactly as its --krylov mode does (checked against the stored goldens) and
writes, per configuration, ml.solve(accel='cgnr' | 'cgne' | 'minimal_residual' | 'steepest_descent') of the reference
(pyamg.krylov, criteria 'rr') with the cycle as preconditioner: iterate, residual list and info of every RUNS entry.
No other golden file is written.
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden  # noqa: E402

# per method: V-cycle from zero to a tight tol, a W- or F-cycle from the stored x0 to a loose tol, and b = 0 from
# x0 = 0 (CGNR / CGNE return at once, minimal residual scales by 1, steepest descent computes 0 / 0)
RUNS = {}
for _m, _c in (("cgnr", "W"), ("cgne", "F"), ("minimal_residual", "W"), ("steepest_descent", "F")):
    RUNS[_m] = dict(tol=1e-10, maxiter=8, accel=_m)
    RUNS[_m + "_x0"] = dict(tol=1e-3, maxiter=20, accel=_m, cycle=_c)
    RUNS[_m + "_zero"] = dict(tol=1e-8, maxiter=4, accel=_m)


def emit_krylov_more(name, ml, b, x0):
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with np.errstate(invalid="ignore"):
            for tag, kw in RUNS.items():
                kw = dict(kw)
                rhs = np.zeros_like(b) if tag.endswith("_zero") else b
                if tag.endswith("_x0"):
                    kw["x0"] = x0
                res = []
                x, info = ml.solve(rhs, residuals=res, return_info=True, **kw)
                out["x_ref_" + tag] = x
                out["residuals_" + tag] = np.array(res)
                out["info_" + tag] = np.array([info])
    os.makedirs(os.path.join(make_golden.HERE, "krylov_more"), exist_ok=True)
    np.savez_compressed(os.path.join(make_golden.HERE, "krylov_more", name + ".npz"), **out)
    print(f"krylov_more/{name}: " + ", ".join(f"{t}: {len(out['residuals_' + t]) - 1} its info={int(out['info_' + t][0])}"
                                            for t in RUNS))


if __name__ == "__main__":
    if "--only" in sys.argv:
        make_golden.ONLY = sys.argv[sys.argv.index("--only") + 1]
    # make_golden's --krylov mode rebuilds every hierarchy, checks it against the stored golden and hands it to
    # emit_krylov; here that hand-off writes the krylov_more fixtures instead
    make_golden.KRYLOV_ONLY = True
    make_golden.emit_krylov = emit_krylov_more
    make_golden.main()
    make_golden.main_widening()
