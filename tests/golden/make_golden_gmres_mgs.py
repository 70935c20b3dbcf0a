"""Generate tests/golden/krylov_mgs/<cfg>.npz by running the REAL reference (see make_golden.py):

    AMGB_REFERENCE=<reference checkout> python oracle/build.py
    PYTHONPATH=oracle/_ref/site python tests/golden/make_golden_gmres_mgs.py

Rebuilds make_golden.py's hierarchies exactly as its --krylov mode does (checked against the stored goldens) and
writes, per configuration, the reference's modified Gram-Schmidt GMRES with the cycle as preconditioner: iterate,
residual list and info of every RUNS entry.  No other golden file is written.
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden  # noqa: E402

# a V-cycle from zero to a tight tol; W and F from the stored x0; b = 0 from the stored x0 (||M b|| is taken as 1);
# reorth=True through pyamg.krylov.gmres_mgs(A, b, M=ml.aspreconditioner()); and a stagnation case: b = A u with
# u = 2 + x0 / max|x0| (no entry near zero), started from (1 + 3e-15) u, so the first update is about 3e-15 x and the
# method stops with info = -1
RUNS = {"mgs": dict(tol=1e-10, maxiter=12),
        "mgsW": dict(tol=1e-3, maxiter=25, cycle="W"),
        "mgsF": dict(tol=1e-4, maxiter=25, cycle="F"),
        "mgs_zero": dict(tol=1e-8, maxiter=6),
        "mgs_reorth": dict(tol=1e-10, maxiter=12),
        "mgs_stag": dict(tol=1e-30, maxiter=3)}
WITH_X0 = ("mgsW", "mgsF", "mgs_zero", "mgs_stag")


def emit_gmres_mgs(name, ml, b, x0):
    from pyamg.krylov import gmres_mgs
    out = {}
    b = np.ravel(b)
    x0 = np.ravel(x0)
    A = ml.levels[0].A
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for tag, kw in RUNS.items():
            kw = dict(kw)
            rhs = b
            if tag == "mgs_zero":
                rhs = np.zeros_like(b)
            if tag in WITH_X0:
                kw["x0"] = x0.copy()
            if tag == "mgs_stag":
                u = 2.0 + x0 / np.max(np.abs(x0))
                rhs = A @ u
                kw["x0"] = u * (1.0 + 3e-15)
                out["b_" + tag] = rhs
                out["x0_" + tag] = kw["x0"].copy()
            res = []
            if tag == "mgs_reorth":
                x, info = gmres_mgs(A, rhs, M=ml.aspreconditioner(cycle="V"), reorth=True, residuals=res, **kw)
            else:
                x, info = ml.solve(rhs, accel="gmres_mgs", residuals=res, return_info=True, **kw)
            out["x_ref_" + tag] = np.ravel(x)
            out["residuals_" + tag] = np.array(res)
            out["info_" + tag] = np.array([info])
    os.makedirs(os.path.join(make_golden.HERE, "krylov_mgs"), exist_ok=True)
    np.savez_compressed(os.path.join(make_golden.HERE, "krylov_mgs", name + ".npz"), **out)
    print(f"krylov_mgs/{name}: " + ", ".join(f"{t}: {len(out['residuals_' + t]) - 1} its info={int(out['info_' + t][0])}"
                                           for t in RUNS))


if __name__ == "__main__":
    if "--only" in sys.argv:
        make_golden.ONLY = sys.argv[sys.argv.index("--only") + 1]
    # make_golden's --krylov mode rebuilds every hierarchy, checks it against the stored golden and hands it to
    # emit_krylov; here that hand-off writes the krylov_mgs fixtures instead
    make_golden.KRYLOV_ONLY = True
    make_golden.emit_krylov = emit_gmres_mgs
    make_golden.main()
    make_golden.main_widening()
