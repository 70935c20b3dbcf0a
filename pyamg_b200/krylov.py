"""Krylov solvers with the call signatures of ``pyamg.krylov`` whose preconditioner is a pyamg_b200 cycle.

The usual way to use the reference's hierarchy as a preconditioner is

    x, info = pyamg.krylov.gmres(A, b, M=ml.aspreconditioner(cycle='V'), tol=1e-8, residuals=res)

which, with a GPU hierarchy behind ``M``, would bounce every Krylov vector host <-> device once per iteration.
The functions below take the same arguments; when ``M`` comes from ``pyamg_b200.MultilevelSolver.aspreconditioner``
and ``A`` is that hierarchy's fine-level operator they run the whole accelerated solve resident in HBM
(``amgb_solve_cg`` / ``amgb_solve_gmres`` / ``amgb_solve_bicgstab``: pyamg/krylov/_cg.py, _gmres_householder.py,
_gmres_mgs.py, _fgmres.py, _bicgstab.py restated, see csrc/abi_krylov.cuh; ``amgb_solve_krylov``: _cgnr.py, _cgne.py,
_minimal_residual.py, _steepest_descent.py, see csrc/abi_krylov_more.cuh).  ``b`` (and ``x0``) may be CUDA tensors: they stay in device memory and x is a CUDA tensor.
Anything else is outside the accelerated path and raises -- there is no CPU fallback here;
SciPy's / the reference's host solvers accept the same ``M`` unchanged.
"""
import numpy as np

from .multilevel import _is_cuda

__all__ = ["cg", "gmres", "gmres_householder", "gmres_mgs", "fgmres", "bicgstab", "cgnr", "cgne", "minimal_residual",
           "steepest_descent"]


def _resident(A, M, name):
    ml = getattr(M, "_amgb_solver", None)
    if ml is None:
        raise NotImplementedError(f"pyamg_b200.krylov.{name}: M must come from pyamg_b200.MultilevelSolver.aspreconditioner "
                                  "(host Krylov solvers accept that operator too)")
    A0 = ml.levels[0].A
    same = A is A0
    if not same and getattr(A, "shape", None) == A0.shape:
        try:
            same = (abs(A - A0)).nnz == 0
        except (TypeError, ValueError):
            same = False
    if not same:
        raise NotImplementedError(f"pyamg_b200.krylov.{name}: A must be the fine-level operator of the preconditioning "
                                  "hierarchy (ml.levels[0].A)")
    return ml, M._amgb_cycle


def _run(name, A, b, x0, tol, maxiter, M, callback, residuals, restart=None, reorth=False):
    if callback is not None:
        raise NotImplementedError(f"pyamg_b200.krylov.{name}: callbacks need host iterates; use ml.solve(accel=...)")
    if restart is not None:
        raise NotImplementedError(f"pyamg_b200.krylov.{name}: restarts are not exposed (amgb_solve_gmres has them)")
    ml, cycle = _resident(A, M, name)
    b = b if _is_cuda(b) else np.asarray(b)      # CUDA tensors stay on the device (MultilevelSolver.solve)
    if reorth:
        # solve() has no reorth argument (nor has the reference's): the resident path is called directly, with
        # solve(accel='gmres_mgs')'s checks
        if ml.levels[0].A.shape[0] < 2 or (not _is_cuda(b) and np.iscomplexobj(b)):
            raise NotImplementedError(f"pyamg_b200.krylov.{name}: reorth=True runs on real systems with n >= 2")
        cycle = ml._check_cycle(cycle, name)
        x, info = ml._solve_resident(name, b, x0, tol, maxiter, cycle, residuals, True, reorth=True)
    else:
        x, info = ml.solve(b, x0=x0, tol=tol, maxiter=maxiter, cycle=cycle, accel=name, residuals=residuals,
                           return_info=True)
    return x.reshape(b.shape), info


def cg(A, b, x0=None, tol=1e-5, criteria="rr", maxiter=None, M=None, callback=None, residuals=None):
    """pyamg.krylov.cg (krylov/_cg.py:11-196) with the cycle ``M``, resident on the GPU (criteria 'rr' only)."""
    if criteria != "rr":
        raise NotImplementedError("pyamg_b200.krylov.cg: stopping criteria 'rr' only")
    return _run("cg", A, b, x0, tol, maxiter, M, callback, residuals)


def gmres(A, b, x0=None, tol=1e-5, restart=None, maxiter=None, M=None, callback=None, residuals=None,
          orthog="householder", **kwargs):
    """pyamg.krylov.gmres (krylov/_gmres.py:11-127 -> _gmres_householder.py, or _gmres_mgs.py for orthog='mgs') with
    the cycle ``M``, resident."""
    if orthog == "mgs":
        return gmres_mgs(A, b, x0=x0, tol=tol, restart=restart, maxiter=maxiter, M=M, callback=callback,
                         residuals=residuals, **kwargs)
    if orthog != "householder":
        raise NotImplementedError("pyamg_b200.krylov.gmres: orthog='householder' (the reference's default) or 'mgs'")
    return _run("gmres", A, b, x0, tol, maxiter, M, callback, residuals, restart)


def fgmres(A, b, x0=None, tol=1e-5, restart=None, maxiter=None, M=None, callback=None, residuals=None, **kwargs):
    """pyamg.krylov.fgmres (krylov/_fgmres.py:17-345) with the cycle ``M``, resident."""
    return _run("fgmres", A, b, x0, tol, maxiter, M, callback, residuals, restart)


def bicgstab(A, b, x0=None, tol=1e-5, criteria="rr", maxiter=None, M=None, callback=None, residuals=None):
    """pyamg.krylov.bicgstab (krylov/_bicgstab.py:10-200) with the cycle ``M``, resident (criteria 'rr' only)."""
    if criteria != "rr":
        raise NotImplementedError("pyamg_b200.krylov.bicgstab: stopping criteria 'rr' only")
    return _run("bicgstab", A, b, x0, tol, maxiter, M, callback, residuals)


def gmres_householder(A, b, x0=None, tol=1e-5, restart=None, maxiter=None, M=None, callback=None, residuals=None,
                      restrt=None):
    """pyamg.krylov.gmres_householder (krylov/_gmres_householder.py:21-360) with the cycle ``M``, resident: what
    ``gmres`` runs."""
    if restrt is not None:
        raise NotImplementedError("pyamg_b200.krylov.gmres_householder: restarts are not exposed")
    return _run("gmres_householder", A, b, x0, tol, maxiter, M, callback, residuals, restart)


def gmres_mgs(A, b, x0=None, tol=1e-5, restart=None, maxiter=None, M=None, callback=None, residuals=None, reorth=False,
              restrt=None):
    """pyamg.krylov.gmres_mgs (krylov/_gmres_mgs.py:42-342) with the cycle ``M``, resident; ``reorth=True`` adds the
    reference's second Gram-Schmidt pass where the projections removed almost all of the new vector."""
    if restrt is not None:
        raise NotImplementedError("pyamg_b200.krylov.gmres_mgs: restarts are not exposed")
    return _run("gmres_mgs", A, b, x0, tol, maxiter, M, callback, residuals, restart,
                reorth=reorth is True)                 # the reference tests `reorth is True` (:260)


def cgnr(A, b, x0=None, tol=1e-5, criteria="rr", maxiter=None, M=None, callback=None, residuals=None):
    """pyamg.krylov.cgnr (krylov/_cgnr.py:12-220) with the cycle ``M``, resident (criteria 'rr' only)."""
    if criteria != "rr":
        raise NotImplementedError("pyamg_b200.krylov.cgnr: stopping criteria 'rr' only")
    return _run("cgnr", A, b, x0, tol, maxiter, M, callback, residuals)


def cgne(A, b, x0=None, tol=1e-5, criteria="rr", maxiter=None, M=None, callback=None, residuals=None):
    """pyamg.krylov.cgne (krylov/_cgne.py:12-214) with the cycle ``M``, resident (criteria 'rr' only)."""
    if criteria != "rr":
        raise NotImplementedError("pyamg_b200.krylov.cgne: stopping criteria 'rr' only")
    return _run("cgne", A, b, x0, tol, maxiter, M, callback, residuals)


def minimal_residual(A, b, x0=None, tol=1e-5, maxiter=None, M=None, callback=None, residuals=None):
    """pyamg.krylov.minimal_residual (krylov/_minimal_residual.py:10-163) with the cycle ``M``, resident."""
    return _run("minimal_residual", A, b, x0, tol, maxiter, M, callback, residuals)


def steepest_descent(A, b, x0=None, tol=1e-5, criteria="rr", maxiter=None, M=None, callback=None, residuals=None):
    """pyamg.krylov.steepest_descent (krylov/_steepest_descent.py:11-197) with the cycle ``M``, resident (criteria
    'rr' only)."""
    if criteria != "rr":
        raise NotImplementedError("pyamg_b200.krylov.steepest_descent: stopping criteria 'rr' only")
    return _run("steepest_descent", A, b, x0, tol, maxiter, M, callback, residuals)
