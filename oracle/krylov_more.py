"""CPU restatement of the reference's CGNR, CGNE, minimal residual and steepest descent.  TEST INFRASTRUCTURE ONLY
(see oracle/__init__.py): the checker of `amgb_solve_krylov`, never imported by the product.

Follows, statement by statement and with criteria 'rr',
  pyamg/krylov/_cgnr.py:97-220               (A^H applied as ``A.T.conjugate() @ r``),
  pyamg/krylov/_cgne.py:97-214,
  pyamg/krylov/_minimal_residual.py:92-163   (residual list = ||M r||; r recomputed on every step but each 50th),
  pyamg/krylov/_steepest_descent.py:92-197   (no stop test before the loop; r recomputed as in minimal residual),
with the norm of pyamg/util/linalg.py:13-55.  ``ml.solve(accel=<name>)`` reaches these through multilevel.py:479-508
with ``M = aspreconditioner(cycle)``; ``run`` drives them with an oracle Cycle as M.

Pinned by tests/test_oracle_more_krylov.py against goldens the real reference produced (tests/golden/krylov_more/,
written by tests/golden/make_golden_krylov_more.py).
"""
from warnings import warn

import numpy as np

from .krylov import _norm

METHODS = ("cgnr", "cgne", "minimal_residual", "steepest_descent")


def _setup(A, b, x0, M):
    if M is None:
        def M(v):
            return v.copy()
    b = np.ravel(np.asarray(b, dtype=np.float64))
    x = np.zeros(len(b)) if x0 is None else np.array(np.ravel(x0), dtype=np.float64)
    return b, x, M


def _cgn_maxiter(maxiter, n):
    """_cgnr.py:109-116 / _cgne.py:109-116 (the clamp's warning is the caller's)."""
    if maxiter is None:
        return int(np.ceil(1.3 * n)) + 2
    if maxiter < 1:
        raise ValueError("Number of iterations must be positive")
    if maxiter > 1.3 * n:
        return int(np.ceil(1.3 * n)) + 2
    return maxiter


def cgnr(A, b, x0=None, tol=1e-5, maxiter=None, M=None, residuals=None):
    AH = A.T.conjugate()
    b, x, M = _setup(A, b, x0, M)
    maxiter = _cgn_maxiter(maxiter, len(b))
    r = b - A @ x
    rhat = AH @ r
    normr = np.linalg.norm(r)
    z = M(rhat)
    p = z.copy()
    old_zr = np.inner(z, rhat)
    if residuals is not None:
        residuals[:] = [normr]
    normb = _norm(b)
    if normb == 0.0:
        normb = 1.0
    rtol = tol * normb
    if normr < rtol:
        return x, 0
    it = 0
    while True:
        w = A @ p
        alpha = old_zr / np.inner(w, w)
        x += alpha * p
        if np.mod(it, 8) and it > 0:
            r -= alpha * w
        else:
            r = b - A @ x
        rhat = AH @ r
        z = M(rhat)
        new_zr = np.inner(z, rhat)
        beta = new_zr / old_zr
        old_zr = new_zr
        p *= beta
        p += z
        it += 1
        normr = np.linalg.norm(r)
        if residuals is not None:
            residuals.append(normr)
        if normr < rtol:
            return x, 0
        if it == maxiter:
            return x, it


def cgne(A, b, x0=None, tol=1e-5, maxiter=None, M=None, residuals=None):
    AH = A.T.conjugate()
    b, x, M = _setup(A, b, x0, M)
    maxiter = _cgn_maxiter(maxiter, len(b))
    r = b - A @ x
    normr = _norm(r)
    z = M(r)
    p = AH @ z
    old_zr = np.inner(z, r)
    if residuals is not None:
        residuals[:] = [normr]
    normb = _norm(b)
    if normb == 0.0:
        normb = 1.0
    rtol = tol * normb
    if normr < rtol:
        return x, 0
    it = 0
    while True:
        alpha = old_zr / np.inner(p, p)
        x += alpha * p
        if np.mod(it, 8) and it > 0:
            r -= alpha * (A @ p)
        else:
            r = b - A @ x
        z = M(r)
        new_zr = np.inner(z, r)
        beta = new_zr / old_zr
        old_zr = new_zr
        p *= beta
        p += AH @ z
        it += 1
        normr = np.linalg.norm(r)
        if residuals is not None:
            residuals.append(normr)
        if normr < rtol:
            return x, 0
        if it == maxiter:
            return x, it


def minimal_residual(A, b, x0=None, tol=1e-5, maxiter=None, M=None, residuals=None):
    b, x, M = _setup(A, b, x0, M)
    if maxiter is None:
        maxiter = int(1.3 * len(b)) + 2
    elif maxiter < 1:
        raise ValueError("Number of iterations must be positive")
    r = b - A @ x
    z = M(r)
    normr = _norm(z)
    if residuals is not None:
        residuals[:] = [normr]
    normb = _norm(b)
    normMb = 1.0 if normb == 0.0 else _norm(M(b))
    if normr < tol * normMb:
        return x, 0
    it = 0
    while True:
        p = M(A @ z)
        pz = np.inner(p, z)
        if pz < 0.0:
            warn("\nIndefinite matrix detected in minimal residual, stopping.\n")
            return x, -1
        alpha = pz / np.inner(p, p)
        x = x + alpha * z
        it += 1
        if np.mod(it, 50) and it > 0:
            r = b - A @ x
            z = M(r)
        else:
            z = z - alpha * p
        normr = _norm(z)
        if residuals is not None:
            residuals.append(normr)
        if normr < tol * normMb:
            return x, 0
        if it == maxiter:
            return x, it


def steepest_descent(A, b, x0=None, tol=1e-5, maxiter=None, M=None, residuals=None):
    b, x, M = _setup(A, b, x0, M)
    if maxiter is None:
        maxiter = len(b)
    elif maxiter < 1:
        raise ValueError("Number of iterations must be positive")
    r = b - A @ x
    z = M(r)
    rz = np.inner(r, z)
    normr = np.linalg.norm(r)
    if residuals is not None:
        residuals[:] = [normr]
    normb = _norm(b)
    if normb == 0.0:
        normb = 1.0
    rtol = tol * normb
    it = 0
    with np.errstate(invalid="ignore"):          # b = 0 from x0 = 0: alpha = 0 / 0, as in the reference
        while True:
            q = A @ z
            zAz = np.inner(z, q)
            if zAz < 0.0:
                warn("\nIndefinite matrix detected in steepest descent, aborting\n")
                return x, -1
            alpha = rz / zAz
            x = x + alpha * z
            it += 1
            if np.mod(it, 50) and it > 0:
                r = b - A @ x
            else:
                r = r - alpha * q
            z = M(r)
            rz = np.inner(r, z)
            if rz < 0.0:
                warn("\nIndefinite preconditioner detected in steepest descent, stopping.\n")
                return x, -1
            normr = _norm(r)
            if residuals is not None:
                residuals.append(normr)
            if normr < rtol:
                return x, 0
            if rz == 0.0:
                warn("\nSingular preconditioner detected in steepest descent, stopping.\n")
                return x, -1
            if it == maxiter:
                return x, it


def run(cyc, method, b, x0=None, tol=1e-5, maxiter=100, cycle="V", residuals=None):
    """``ml.solve(b, accel=method, ...)`` of the reference with the oracle Cycle ``cyc`` as the preconditioner
    (one cycle from zero, multilevel.py:390-396)."""
    fn = {"cgnr": cgnr, "cgne": cgne, "minimal_residual": minimal_residual,
          "steepest_descent": steepest_descent}[method]
    A0 = cyc.levels[0]["A"]
    return fn(A0, b, x0=x0, tol=tol, maxiter=maxiter, residuals=residuals,
              M=lambda r: cyc.solve(r, maxiter=1, cycle=cycle, tol=1e-12))
