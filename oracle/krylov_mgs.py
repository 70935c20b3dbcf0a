"""CPU restatement of the reference's modified Gram-Schmidt GMRES.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py):
the checker of ``amgb_solve_gmres`` with ``AMGB_FLAG_MGS``, never imported by the product.

Follows pyamg/krylov/_gmres_mgs.py:42-342 statement by statement: LEFT preconditioning, stop on the preconditioned
residual against ||M b|| (1 when b = 0), Givens rotations from LAPACK lartg, the optional second Gram-Schmidt pass
(``reorth``) and the stagnation test.  ``ml.solve(accel='gmres_mgs')`` reaches it through multilevel.py:479-508 with
``M = aspreconditioner(cycle)`` (one cycle from a zero guess).

Pinned by tests/test_oracle_gmres_mgs.py against goldens the real reference produced (tests/golden/krylov_mgs/).
"""
import warnings

import numpy as np
import scipy.linalg
from scipy.linalg import get_lapack_funcs

from oracle.krylov import _norm


def gmres_mgs(A, b, x0=None, tol=1e-5, restart=None, maxiter=None, M=None, residuals=None, reorth=False,
              matvec=None):
    """``M`` and ``matvec`` are callables (v -> M v, A v); by default ``matvec`` is ``A @ v`` and M the identity."""
    if matvec is None:
        def matvec(v):
            return A @ v
    if M is None:
        def M(v):
            return v.copy()
    b = np.ravel(np.asarray(b, dtype=np.float64))
    n = len(b)
    x = np.zeros(n) if x0 is None else np.array(np.ravel(x0), dtype=np.float64)
    [lartg] = get_lapack_funcs(["lartg"], [x])

    # outer / inner iteration limits (:168-185)
    if restart:
        max_outer = maxiter if maxiter else 1
        if restart > n:
            warnings.warn("Setting restart to maximum allowed, n.")
            restart = n
        max_inner = restart
    else:
        max_outer = 1
        if maxiter is None:
            maxiter = min(n, 40)
        elif maxiter > n:
            warnings.warn("Setting maxiter to maximum allowed, n.")
            maxiter = n
        max_inner = maxiter
    if n == 1:
        entry = np.ravel(matvec(np.array([1.0])))
        return b / entry, 0

    r = np.ravel(M(b - matvec(x)))
    normr = _norm(r)
    if residuals is not None:
        residuals[:] = [normr]
    normMb = 1.0 if _norm(b) == 0.0 else _norm(M(b))
    if normr < tol * normMb:
        return x, 0
    niter = 0

    for _outer in range(max_outer):
        Q = []                                          # Givens rotations, appended when formed
        H = np.zeros((max_inner + 1, max_inner + 1))    # row `inner` holds the Hessenberg column `inner`
        V = np.zeros((max_inner + 1, n))                # Krylov basis, one vector per row
        V[0, :] = r * (1.0 / normr)
        g = np.zeros(n)
        g[0] = normr

        for inner in range(max_inner):
            v = V[inner + 1, :]
            v[:] = np.ravel(M(matvec(V[inner, :])))
            normv_old = _norm(v)
            for k in range(inner + 1):                  # modified Gram-Schmidt: project, then update, in turn
                alpha = np.dot(V[k, :], v)
                H[inner, k] = alpha
                v -= alpha * V[k, :]
            normv = _norm(v)
            H[inner, inner + 1] = normv
            if reorth is True and normv_old == normv_old + 0.001 * normv:
                for k in range(inner + 1):
                    alpha = np.dot(V[k, :], v)
                    H[inner, k] = H[inner, k] + alpha
                    v -= alpha * V[k, :]
            if H[inner, inner + 1] != 0.0:
                v *= 1.0 / H[inner, inner + 1]
            for j in range(inner):                      # the earlier rotations on the new column
                H[inner, j:j + 2] = np.dot(Q[j], H[inner, j:j + 2])
            if inner != n - 1 and H[inner, inner + 1] != 0:
                c, s, _r = lartg(H[inner, inner], H[inner, inner + 1])
                Qblock = np.array([[c, s], [-s, c]])
                Q.append(Qblock)
                g[inner:inner + 2] = np.dot(Qblock, g[inner:inner + 2])
                H[inner, inner] = np.dot(Qblock[0, :], H[inner, inner:inner + 2])
                H[inner, inner + 1] = 0.0
            niter += 1
            if inner < max_inner - 1:                   # the converged estimate is never recorded
                normr = np.abs(g[inner + 1])
                if normr < tol * normMb:
                    break
                if residuals is not None:
                    residuals.append(normr)

        y = scipy.linalg.solve(H[0:inner + 1, 0:inner + 1].T, g[0:inner + 1])
        update = np.ravel(V[:inner + 1, :].T.dot(y.reshape(-1, 1)))
        x = x + update
        r = np.ravel(M(b - matvec(x)))
        normr = _norm(r)
        if residuals is not None:
            residuals.append(normr)
        indices = x != 0
        if indices.any():
            change = np.max(np.abs(update[indices] / x[indices]))
            if change < 1e-12:
                return x, -1
        if normr < tol * normMb:
            return x, 0

    return x, niter


def run(cyc, b, x0=None, tol=1e-5, maxiter=100, cycle="V", residuals=None, reorth=False, restart=None):
    """``ml.solve(b, accel='gmres_mgs', ...)`` of the reference (``reorth=True``: ``pyamg.krylov.gmres_mgs(A, b,
    M=ml.aspreconditioner(cycle), reorth=True, ...)``) with the oracle Cycle ``cyc`` as the preconditioner."""
    A0 = cyc.levels[0]["A"]
    return gmres_mgs(A0, b, x0=x0, tol=tol, restart=restart, maxiter=maxiter, residuals=residuals, reorth=reorth,
                     M=lambda r: cyc.solve(r, maxiter=1, cycle=cycle, tol=1e-12))
