"""MultilevelSolver: the reference's hierarchy container and cycle API, executed on an H100.

Mirror of pyamg/multilevel.py.  The object API is kept (``levels`` list of ``Level`` structs with
``A, P, R, presmoother, postsmoother``; ``solve`` :398-582 with the same keyword arguments, return
values and stop test; ``aspreconditioner`` :355-396; ``psolve``; ``change_solve_matrix``;
``__repr__`` and the three complexity measures :184-318), but ``solve`` no longer recurses through
NumPy/SciPy: the hierarchy is uploaded once to HBM and the cycle (pre-smooth, residual,
restriction, coarse solve, prolongation + correction, post-smooth) runs as sm_90a CUDA kernels
captured in a CUDA graph (csrc/engine.cu).  Host arrays in, a new host array out -- or CUDA tensors in and a
CUDA tensor out, with every vector kept in device memory (``solve`` / ``solve_many`` on ``torch.Tensor`` inputs).

Build it from
  * a reference solver:  ``MultilevelSolver.from_pyamg(pyamg.ruge_stuben_solver(A))``
    (setup stays on the reference's CPU path; closures are parsed for omega / Dinv / row lists), or
  * a list of ``Level`` objects exactly as the reference's constructors do, followed by
    ``pyamg_b200.relaxation.smoothing.change_smoothers``.

No CPU fallback: without libpyamg_b200.so and a CUDA device ``solve`` raises.
"""
import ctypes
import os
import sys
import warnings
from dataclasses import dataclass
from warnings import warn

import numpy as np
import scipy.linalg
import scipy.sparse.linalg as sla
from scipy import sparse
from scipy.sparse.linalg import LinearOperator

from . import _engine as E
from .relaxation import smoothing

__all__ = ["MultilevelSolver", "coarse_grid_solver"]


def coarse_solver_spec(cs):
    """The ``coarse_solver=`` argument a coarse solver object was built from: ``name`` or ``(name, kwargs)``.

    The reference's ``GenericSolver.name()`` returns only the method name (multilevel.py:820-823); its keyword
    arguments -- e.g. the sweep count of a relaxation coarse solver -- live in the closure of the ``solve`` function
    its ``__call__`` uses (:700-790).  They are read from there, so that a reference-built hierarchy is adopted with
    the coarse solver it really has."""
    import ast
    own = getattr(cs, "spec", None)
    if own is not None:
        return own
    name = cs.name() if hasattr(cs, "name") else "'pinv'"
    try:
        name = ast.literal_eval(name)
    except (ValueError, SyntaxError) as exc:
        raise NotImplementedError(f"coarse solver {name} is not on the GPU hot path") from exc
    kwargs = {}
    try:
        call = type(cs).__call__
        cells = dict(zip(call.__code__.co_freevars, [c.cell_contents for c in call.__closure__ or ()]))
        solve = cells.get("solve")
        if solve is not None and solve.__closure__:
            kwargs = dict(zip(solve.__code__.co_freevars, [c.cell_contents for c in solve.__closure__])).get("kwargs", {})
    except (AttributeError, TypeError, ValueError):
        kwargs = {}
    if isinstance(name, tuple):
        return name
    return (name, dict(kwargs)) if kwargs else name


def _is_cuda(v):
    """Whether v is a torch CUDA tensor.  torch is looked up, not imported: importing pyamg_b200 does not import it,
    and a caller holding a tensor has imported it already."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(v, torch.Tensor) and v.is_cuda


def _ptr(a):
    """Address of a host array's or a CUDA tensor's first element, for the engine's C entry points."""
    return a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr()


def _new_block(B, X0, dev, zero=False):
    """The (n, k) float64 block solve_many's engine call writes: a copy of X0 (which is never written), else new
    (zeros if `zero`); a C-contiguous array, or a contiguous tensor on B's device."""
    if dev:
        torch = sys.modules["torch"]
        if X0 is not None:
            return X0.clone()
        return (torch.zeros if zero else torch.empty)(tuple(B.shape), dtype=torch.float64, device=B.device)
    if X0 is not None:
        return np.array(X0, dtype=np.float64, order="C")
    return np.zeros(B.shape) if zero else np.empty(B.shape)


@dataclass(frozen=True)
class _Accel:
    """A GPU-resident accelerator: the reference's pyamg.krylov function ``name`` (criteria 'rr') with one cycle from
    zero as M, run on one vector by ``amgb_solve_<entry>`` and on k columns by ``amgb_solve_many_<entry>``."""
    name: str
    entry: str                      # "cg", "bicgstab", "gmres", or "krylov" (method E.KRYLOV[name])
    default_maxiter: object = None  # n -> the iterations of maxiter=None; the GMRES family takes min(n, 40) steps
    min_n: int = 1                  # fewest unknowns the engine takes; smaller systems run a host solver
    flags: int = 0                  # E.FLAG_FLEXIBLE, E.FLAG_MGS
    clamp: str = None               # CGNR / CGNE: warned when maxiter > 1.3 n is cut to the default
    stop: object = None             # warning for info = -1: one text, or a text per reason the engine reports
                                    # (none for CGNR / CGNE)
    transpose: bool = False         # needs A^H of the fine level on the device (MultilevelSolver._transpose0)

    def iterations(self, maxiter, n):
        """(maxiter for the engine, rows of the residual buffer, clamp warning or None): the reference's default and
        check of maxiter (_cg.py:92-93, _bicgstab.py:90-91, _gmres_householder.py:146-148, _gmres_mgs.py:182,
        _cgnr.py:109-116, _cgne.py:109-116, _minimal_residual.py:101-104, _steepest_descent.py:98-101)."""
        if self.entry == "gmres":   # the engine cuts maxiter to n; max_inner + 3 residuals at most
            max_inner = min(n, 40) if maxiter is None else min(int(maxiter), n)
            clamp = "Setting maxiter to maximum allowed, n." if maxiter is not None and maxiter > n else None
            return (0 if maxiter is None else int(maxiter)), max_inner + 3, clamp
        if maxiter is not None and maxiter < 1:
            raise ValueError("Number of iterations must be positive")
        if maxiter is None or (self.clamp is not None and maxiter > 1.3 * n):
            its = self.default_maxiter(n)
            return its, its + 1, None if maxiter is None else self.clamp
        return int(maxiter), int(maxiter) + 1, None

    def stop_warnings(self, info, reason):
        """The texts warned for the columns that stopped with info = -1, each once."""
        if self.stop is None or not (info == -1).any():
            return []
        if isinstance(self.stop, str):
            return [self.stop]
        return [self.stop[why] for why in sorted(set(reason[info == -1].tolist()))]

    def call(self, h, k, b, x, tol, maxiter, cycle, flags, res, nres, info, reason):
        """The engine call on one vector (k None) or on k columns; returns its status code."""
        fn = getattr(E.lib(), ("amgb_solve_" if k is None else "amgb_solve_many_") + self.entry)
        cols = () if k is None else (k,)
        args = (b, x, float(tol))
        tail = (E.i32p(nres), E.i32p(info))
        resp = None if res is None else E.f64p(res)
        flags |= self.flags
        if self.entry == "gmres":
            return fn(h, *cols, *args, 0, int(maxiter), cycle, flags, resp, res.shape[0], *tail)
        if self.entry == "krylov":
            return fn(h, E.KRYLOV[self.name], *cols, *args, int(maxiter), cycle, flags, resp, *tail, E.i32p(reason))
        return fn(h, *cols, *args, int(maxiter), cycle, flags, resp, *tail)


_CG_STOP = "\nIndefinite matrix or preconditioner detected in CG, aborting\n"
_GMRES = _Accel("gmres", "gmres", min_n=2)
# the resident accelerators by the names solve(accel=...) takes, with the reference's texts as it spells them
_ACCELS = {
    "cg": _Accel("cg", "cg", lambda n: int(1.3 * n) + 2, stop=_CG_STOP),
    "bicgstab": _Accel("bicgstab", "bicgstab", lambda n: n + 5, min_n=2, stop=_CG_STOP),
    "gmres": _GMRES,
    "gmres_householder": _GMRES,    # what the reference resolves both names to
    "gmres_mgs": _Accel("gmres_mgs", "gmres", min_n=2, flags=E.FLAG_MGS),
    "fgmres": _Accel("fgmres", "gmres", min_n=2, flags=E.FLAG_FLEXIBLE),
    "cgnr": _Accel("cgnr", "krylov", lambda n: int(np.ceil(1.3 * n)) + 2, transpose=True, stop={}, clamp=(
        "maximum allowed inner iterations (maxiter) are the 130% times               the number of dofs")),
    "cgne": _Accel("cgne", "krylov", lambda n: int(np.ceil(1.3 * n)) + 2, transpose=True, stop={},
                   clamp="maximum allowed inner iterations (maxiter) are the 130% timesthe number of dofs"),
    "minimal_residual": _Accel("minimal_residual", "krylov", lambda n: int(1.3 * n) + 2, stop={
        E.REASON_INDEFINITE_MATRIX: "\nIndefinite matrix detected in minimal residual, stopping.\n"}),
    "steepest_descent": _Accel("steepest_descent", "krylov", lambda n: n, stop={
        E.REASON_INDEFINITE_MATRIX: "\nIndefinite matrix detected in steepest descent, aborting\n",
        E.REASON_INDEFINITE_PRECONDITIONER: "\nIndefinite preconditioner detected in steepest descent, stopping.\n",
        E.REASON_SINGULAR_PRECONDITIONER: "\nSingular preconditioner detected in steepest descent, stopping.\n"}),
}
_ACCEL_NAMES = ", ".join(map(repr, list(_ACCELS)[:-1])) + f" and {list(_ACCELS)[-1]!r}"
_SPD_WARNING = ("Incompatible non-symmetric multigrid preconditioner detected, due to presmoother/postsmoother "
                "combination. CG requires SPD preconditioner, not just SPD matrix.")


def _resident(accel):
    """The table entry of an accel name, or None."""
    return _ACCELS.get(accel) if isinstance(accel, str) else None


# relaxation methods usable as the coarsest-level solver (multilevel.py:764-766) that the engine runs
_RELAXATION_COARSE = ("gauss_seidel", "jacobi", "block_gauss_seidel", "schwarz", "block_jacobi", "richardson", "sor",
                      "chebyshev", "jacobi_ne", "gauss_seidel_ne", "gauss_seidel_nr")


def coarse_grid_solver(solver):
    """Coarse-level solver descriptor (pyamg/multilevel.py:665-826).

    The engine applies the coarsest solve as a dense matrix-vector product with a matrix computed
    once on the CPU: the pseudo-inverse for 'pinv'/'pinv2' (what the reference caches, :717-721),
    the plain inverse for the direct methods 'lu'/'cholesky'/'splu' (same solve, different
    rounding).  Relaxation methods (:764-781: x = 0, then `iterations` sweeps, default 10) run as the engine's
    smoother kernels on the coarsest level.  Krylov coarse solvers are outside the accelerated path.
    """
    def unpack_arg(v):
        if isinstance(v, tuple):
            return v[0], v[1]
        return v, {}

    name, kwargs = unpack_arg(solver)
    if name in ("pinv", "pinv2"):
        def dense(A):
            return scipy.linalg.pinv(A.toarray(), **kwargs)
    elif name in ("lu", "cholesky", "splu"):
        def dense(A):
            return scipy.linalg.inv(A.toarray())
    elif name is None:
        def dense(A):
            return np.zeros(A.shape)
    elif name in _RELAXATION_COARSE:
        dense = None                                  # x = 0, then `iterations` (default 10) sweeps on the GPU
        kwargs = dict(kwargs)
        kwargs.setdefault("iterations", 10)           # multilevel.py:768-769
    elif isinstance(name, str) or callable(name):
        raise NotImplementedError(f"coarse solver {name!r} is not on the GPU hot path; use 'pinv' "
                                  "(the reference's default), 'lu', 'cholesky', 'splu', a relaxation method "
                                  f"({', '.join(_RELAXATION_COARSE)}) or None")
    else:
        raise ValueError(f"unknown solver: {name}")

    relax_spec = (name, kwargs) if dense is None else None
    relax_name = name                                 # (`name` itself is shadowed inside the class body below)

    class GenericSolver:
        """Holds the cached dense operator (or the relaxation descriptor); applied on the GPU by the cycle engine."""
        relaxation = relax_spec
        spec = solver                                 # what this object was built from (see coarse_solver_spec)
        if relax_spec is not None:
            P = None                                  # no dense operator: the solve is `iterations` GPU sweeps

        def smoother(self, A):
            """The closure the reference builds for a relaxation coarse solver (multilevel.py:773-776)."""
            lvl = MultilevelSolver.Level()
            lvl.A = A
            return smoothing._setup_call(relax_name)(lvl, **kwargs)

        def dense_operator(self, A):
            if not hasattr(self, "P"):
                self.P = np.ascontiguousarray(dense(A), dtype=np.float64)
            return self.P

        def __repr__(self):
            return "coarse_grid_solver(" + repr(solver) + ")"

        @classmethod
        def name(cls):
            return repr(solver)

    return GenericSolver()


def _cg_host(A, b, x0=None, tol=1e-5, maxiter=None, M=None, callback=None, residuals=None):
    """pyamg.krylov.cg (pyamg/krylov/_cg.py:11-196, criteria 'rr') on the host -- the path taken when a
    callback needs host iterates; ``M`` is the GPU cycle as a LinearOperator.  Same steps as amgb_solve_cg."""
    b = np.ravel(np.asarray(b, dtype=np.float64))
    n = len(b)
    x = np.zeros(n) if x0 is None else np.array(np.ravel(x0), dtype=np.float64)
    if maxiter is None:
        maxiter = int(1.3 * n) + 2
    elif maxiter < 1:
        raise ValueError("Number of iterations must be positive")
    r = b - A @ x
    z = M @ r
    p = z.copy()
    rz = np.inner(r, z)
    normr = np.linalg.norm(r)
    if residuals is not None:
        residuals[:] = [normr]
    normb = np.linalg.norm(b)
    if normb == 0.0:
        normb = 1.0
    rtol = tol * normb
    if normr < rtol:
        return x, 0
    it = 0
    while True:
        Ap = A @ p
        rz_old = rz
        pAp = np.inner(Ap, p)
        if pAp < 0.0:
            warn("\nIndefinite matrix detected in CG, aborting\n")
            return x, -1
        alpha = rz / pAp
        x += alpha * p
        if np.mod(it, 8) and it > 0:
            r -= alpha * Ap
        else:
            r = b - A @ x
        z = M @ r
        rz = np.inner(r, z)
        if rz < 0.0:
            warn("\nIndefinite preconditioner detected in CG, aborting\n")
            return x, -1
        beta = rz / rz_old
        p *= beta
        p += z
        it += 1
        normr = np.linalg.norm(r)
        if residuals is not None:
            residuals.append(normr)
        if callback is not None:
            callback(x)
        if normr < rtol:
            return x, 0
        if it == maxiter:
            return x, it


class MultilevelSolver:
    """Stores a multigrid hierarchy and runs the multigrid cycle on the GPU.

    Parameters and attributes as pyamg.multilevel.MultilevelSolver (multilevel.py:17-182).
    """

    class Level:
        """One level of the hierarchy: a struct with A (+ P, R, presmoother, postsmoother)."""

        def __init__(self):
            self.A = None

    def __init__(self, levels, coarse_solver="pinv", device=0, stream=None):
        self.symmetric_smoothing = False
        self.levels = levels
        self.coarse_solver = coarse_grid_solver(coarse_solver)
        self.device = device
        self._stream = stream
        self._h = None
        for level in levels[:-1]:
            if not hasattr(level, "R"):
                level.R = level.P.T.conjugate()     # multilevel.py:180-182

    # ------------------------------------------------------------------ construction helpers
    @classmethod
    def from_pyamg(cls, ml, device=0, stream=None):
        """Adopt a hierarchy built by the reference (any ``pyamg`` constructor): same Level
        objects, same smoother closures, same coarse solver kind (and its cached pinv if any)."""
        spec = coarse_solver_spec(ml.coarse_solver)
        new = cls(list(ml.levels), coarse_solver=spec, device=device, stream=stream)
        new.symmetric_smoothing = getattr(ml, "symmetric_smoothing", False)
        cached = getattr(ml.coarse_solver, "P", None)
        if cached is not None:
            new.coarse_solver.P = np.ascontiguousarray(cached, dtype=np.float64)
        return new

    def _invalidate(self):
        """Drop the device copy (levels or smoothers changed); re-uploaded on the next solve."""
        if self._h is not None:
            E.lib().amgb_hierarchy_destroy(self._h)
            self._h = None
        self._has_transpose0 = False         # A^H went with the device copy (amgb_hierarchy_set_transpose0)

    def __del__(self):
        try:
            self._invalidate()
        except Exception:
            pass

    def upload(self):
        """Upload the hierarchy to HBM (idempotent). Returns the device footprint in bytes."""
        if self._h is not None:
            return int(E.lib().amgb_hierarchy_device_bytes(self._h))
        E.require_gpu()
        L = E.lib()
        h = ctypes.c_void_p()
        E.check(L.amgb_hierarchy_create(int(self.device), ctypes.byref(h)))
        try:
            nlv = len(self.levels)
            for k, lvl in enumerate(self.levels):
                keep = []
                A = E.as_matrix(lvl.A, keep)
                if k < nlv - 1:
                    P = E.as_matrix(lvl.P, keep)
                    R = E.as_matrix(lvl.R, keep)
                    pre = smoothing.describe(getattr(lvl, "presmoother", None), lvl.A, keep)
                    post = smoothing.describe(getattr(lvl, "postsmoother", None), lvl.A, keep)
                    E.check(L.amgb_hierarchy_add_level(h, ctypes.byref(A), ctypes.byref(P),
                                                       ctypes.byref(R), ctypes.byref(pre),
                                                       ctypes.byref(post)))
                else:
                    E.check(L.amgb_hierarchy_add_level(h, ctypes.byref(A), None, None, None, None))
            Ac = self.levels[-1].A
            if Ac.nnz == 0:     # GenericSolver.__call__, multilevel.py:801-803
                E.check(L.amgb_hierarchy_set_coarse_pinv(h, Ac.shape[0], None, 1))
            elif getattr(self.coarse_solver, "relaxation", None) is not None:
                keep = []
                S = smoothing.describe(self.coarse_solver.smoother(Ac), Ac, keep)
                E.check(L.amgb_hierarchy_set_coarse_relaxation(h, ctypes.byref(S)))
            else:
                Pd = self.coarse_solver.dense_operator(Ac)
                E.check(L.amgb_hierarchy_set_coarse_pinv(h, Ac.shape[0], E.f64p(Pd.reshape(-1)), 0))
            E.check(L.amgb_hierarchy_finalize(h, ctypes.c_void_p(self._stream or 0)))
        except Exception:
            L.amgb_hierarchy_destroy(h)
            raise
        self._h = h
        return int(L.amgb_hierarchy_device_bytes(h))

    @property
    def handle(self):
        self.upload()
        return self._h

    def last_launches(self):
        """CUDA kernels launched by the most recent solve (graph nodes counted individually)."""
        return int(E.lib().amgb_hierarchy_last_launches(self._h)) if self._h is not None else 0

    def profile_cycle(self, cycle="V", max_records=200000):
        """Time every operator launch of one (un-graphed) cycle with CUDA events.

        Returns a float array (n, 6): level, op (0 spmv/restrict, 1 residual, 2 prolong+add, 3 jacobi,
        4 gs wave, 5 block jacobi, 6 cluster tail, 7 resident GS, 8 indexed Jacobi, 9 block GS wave, 12 a
        sweep's last gs wave that also writes its rows' residual), rows, nnz,
        algorithmic bytes, milliseconds."""
        rec = np.empty(max_records * 6, dtype=np.float64)
        nrec = ctypes.c_int32(0)
        E.check(E.lib().amgb_profile_cycle(self.handle, E.CYCLES[str(cycle).upper()], E.f64p(rec),
                                           int(max_records), ctypes.byref(nrec)))
        return rec[:nrec.value * 6].reshape(-1, 6).copy()

    # ------------------------------------------------------------------ reporting (host only)
    def __repr__(self):
        """Basic statistics of the hierarchy (multilevel.py:184-209)."""
        output = "MultilevelSolver\n"
        output += f"Number of Levels:     {len(self.levels)}\n"
        output += f"Operator Complexity:  {self.operator_complexity():6.3f}\n"
        output += f"Grid Complexity:      {self.grid_complexity():6.3f}\n"
        output += f"Coarse Solver:        {self.coarse_solver.name()}\n"
        total_nnz = sum(level.A.nnz for level in self.levels)
        output += "  level   unknowns     nonzeros\n"
        for n, level in enumerate(self.levels):
            A = level.A
            ratio = 100 * A.nnz / total_nnz
            output += f"{n:>6} {A.shape[1]:>11} {A.nnz:>12} [{ratio:2.2f}%]\n"
        return output

    def cycle_complexity(self, cycle="V"):
        """Nonzeros touched by one cycle relative to the fine level (multilevel.py:211-283): every visit
        of a non-coarsest level costs 2 nnz (pre + post smoothing), a coarse solve nnz of the coarsest level;
        V visits each level once, W twice per parent visit, F = one F-visit plus one V-visit of the next level."""
        cycle = str(cycle).upper()
        if cycle not in ("V", "W", "F", "AMLI"):
            raise TypeError(f"Unrecognized cycle type ({cycle})")
        nnz = [level.A.nnz for level in self.levels]
        if len(nnz) == 1:
            return 1.0
        # bottom-up: cost of one visit of level l under each recursion pattern
        v = w = f = 2 * nnz[-2] + nnz[-1]
        for l in range(len(nnz) - 3, -1, -1):
            v, w, f = 2 * nnz[l] + v, 2 * nnz[l] + 2 * w, 2 * nnz[l] + f + v
        flops = {"V": v, "W": w, "AMLI": w, "F": f}[cycle]
        return float(flops) / float(nnz[0])

    def operator_complexity(self):
        return sum(level.A.nnz for level in self.levels) / float(self.levels[0].A.nnz)

    def grid_complexity(self):
        return sum(level.A.shape[0] for level in self.levels) / float(self.levels[0].A.shape[0])

    # ------------------------------------------------------------------ solve-phase API
    def change_solve_matrix(self, A):
        """Change the fine-level matrix and rebuild its smoothers (multilevel.py:320-337).

        Levels 1 and below and the coarse solver stay as they were, as in the reference.  When the hierarchy is on
        the device, only level 0 is replaced there (amgb_hierarchy_replace_level0) and the rest stays resident: a
        matrix with the same sparsity pattern, whose rebuilt smoothers differ only in omega, Dinv or coefficients,
        has its values refreshed in place (``_last_replace_path == 1``); anything else rebuilds level 0 alone (2).
        A one-level hierarchy, or a level 0 the engine cannot take, is uploaded again on the next solve (0).  Either
        way every later solve returns what a hierarchy uploaded from scratch on the same levels returns."""
        self.levels[0].A = A
        smoothing.rebuild_smoother(self.levels[0])
        self._last_replace_path = 0
        if self._h is None:
            return
        if len(self.levels) < 2:
            self._invalidate()
            return
        lvl = self.levels[0]
        keep = []
        try:
            M = E.as_matrix(lvl.A, keep)
            pre = smoothing.describe(getattr(lvl, "presmoother", None), lvl.A, keep)
            post = smoothing.describe(getattr(lvl, "postsmoother", None), lvl.A, keep)
        except (NotImplementedError, ValueError, TypeError):
            self._invalidate()              # the next upload reports it, as it did before
            return
        path = ctypes.c_int32(0)
        rc = E.lib().amgb_hierarchy_replace_level0(self._h, ctypes.byref(M), ctypes.byref(pre), ctypes.byref(post),
                                                   None, ctypes.byref(path))
        self._has_transpose0 = False         # the engine dropped A^H of the old matrix
        if rc in (E.ENOTIMPL, E.EINVAL):     # nothing changed on the device: upload from scratch next time
            self._invalidate()
            return
        if rc != E.OK:
            msg = E.lib().amgb_last_error().decode("utf8", "replace")
            self._invalidate()
            raise E.EngineError("change_solve_matrix: " + msg)
        self._last_replace_path = path.value

    # ------------------------------------------------------------------ CUDA tensors (AMGB_FLAG_DEVICE_IO)
    def _device_operand(self, v, name):
        """A CUDA tensor on this hierarchy's device as a contiguous float64 tensor: v itself when it is one, else a
        conversion on the device (as the host path converts with np.ascontiguousarray(..., dtype=float64))."""
        torch = sys.modules["torch"]
        if not _is_cuda(v):
            raise ValueError(f"{name} must be a CUDA tensor, like the other operands of this solve")
        if v.device.index != int(self.device):
            raise ValueError(f"{name} is on {v.device}; this hierarchy is on cuda:{int(self.device)}")
        if v.is_complex():
            raise NotImplementedError("complex systems are outside the fp64 hot path")
        return v.to(torch.float64).contiguous()

    def _device_io(self):
        """AMGB_FLAG_DEVICE_IO for the next engine call, ordered against the caller's current stream: the engine
        reads the operands after the work enqueued there so far, and work enqueued there later sees its result."""
        torch = sys.modules["torch"]
        stream = torch.cuda.current_stream(int(self.device)).cuda_stream
        E.check(E.lib().amgb_hierarchy_set_io_stream(self.handle, stream or E.CUDA_STREAM_LEGACY))
        return E.FLAG_DEVICE_IO

    def _device_vectors(self, b, x0, out=None):
        """b, x and flags of a single-vector engine call on CUDA tensors: b as _device_operand makes it, x = out
        or a new float64 tensor of n entries, holding a copy of x0 (which is never written)."""
        torch = sys.modules["torch"]
        n = self.levels[0].A.shape[0]
        bd = self._device_operand(b, "b").reshape(-1)
        x0d = None if x0 is None else self._device_operand(x0, "x0").reshape(-1)
        if bd.numel() != n or (x0d is not None and x0d.numel() != n):
            raise ValueError("b / x0 have invalid dimensions")
        if out is None:
            xd = torch.empty(n, dtype=torch.float64, device=bd.device)
        elif _is_cuda(out) and out.dtype == torch.float64 and out.is_contiguous() and out.numel() == n \
                and out.device == bd.device:
            xd = out.view(-1)
        else:
            raise ValueError("out must be a contiguous float64 CUDA tensor on the hierarchy's device with as many "
                             "entries as b")
        if x0d is not None:
            xd.copy_(x0d)
        return bd, xd, self._device_io() | (E.FLAG_X0_ZERO if x0 is None else 0)

    def _check_cycle(self, cycle, accel):
        """solve()'s checks of cycle and accel (multilevel.py:472-490) and its CG warning; returns the cycle name."""
        A = self.levels[0].A
        cycle = str(cycle).upper()

        if cycle not in E.CYCLES:
            raise TypeError(f"Unrecognized cycle type ({cycle})")      # :658
        # AMLI cycles require a hermitian matrix (multilevel.py:472-476)
        if cycle == "AMLI" and hasattr(A, "symmetry") and A.symmetry != "hermitian":
            raise ValueError("AMLI cycles require symmetry to be hermitian")

        if accel is not None:
            if accel != "fgmres" and cycle == "AMLI":                  # multilevel.py:487-490
                raise ValueError("AMLI cycles require acceleration (accel) to be fgmres, or no acceleration")
            # Check for symmetric smoothing scheme when using CG (multilevel.py:481-485)
            if (accel == "cg") and (not self.symmetric_smoothing):
                warn(_SPD_WARNING)
        return cycle

    def _solve_resident(self, accel, b, x0, tol, maxiter, cycle, residuals, return_info, reorth=False):
        """solve(accel=accel) on the GPU for an accelerator of _ACCELS, on host arrays or CUDA tensors: the reference's
        function of that name with its maxiter default, clamp and warnings; ``reorth`` is gmres_mgs's option."""
        spec = _ACCELS[accel]
        n = self.levels[0].A.shape[0]
        dev = _is_cuda(b) or _is_cuda(x0)
        if not dev:
            b = np.asarray(b)
            if b.size != n or (x0 is not None and np.asarray(x0).size != n):
                raise ValueError("b / x0 have invalid dimensions")
        its, rows, clamp = spec.iterations(maxiter, n)
        if dev:
            bh, xh, flags = self._device_vectors(b, x0)
        else:
            bh = np.ascontiguousarray(np.ravel(b), dtype=np.float64)
            xh = np.zeros(n) if x0 is None else np.array(np.ravel(x0), dtype=np.float64)
            flags = E.FLAG_X0_ZERO if x0 is None else 0
        if clamp is not None:
            warn(clamp)
        if spec.transpose:
            self._transpose0()
        res = np.empty(rows, dtype=np.float64)
        nres, info, reason = (np.zeros(1, dtype=np.int32) for _ in range(3))
        E.check(spec.call(self.handle, None, _ptr(bh), _ptr(xh), tol, its, E.CYCLES[cycle],
                          flags | (E.FLAG_REORTH if reorth else 0), res, nres, info, reason))
        for text in spec.stop_warnings(info, reason):
            warn(text)
        if residuals is not None:
            residuals[:] = list(res[:nres[0]])
        xout = xh.ravel()          # the reference's Krylov solvers hand back the ravelled iterate
        return (xout, int(info[0])) if return_info else xout

    def _transpose0(self):
        """Upload A^H of the fine level for CGNR / CGNE on their first call on this device copy of the hierarchy
        (change_solve_matrix drops A^H of the old matrix).  Row i holds column i of A in ascending row order of
        A, the order SciPy sums the reference's ``A.T.conjugate() @ r`` in."""
        h = self.handle
        if getattr(self, "_has_transpose0", False):
            return
        AH = sparse.csr_matrix(self.levels[0].A).T.conjugate().tocsr()
        AH.sort_indices()
        keep = []
        M = E.as_matrix(AH, keep)
        E.check(E.lib().amgb_hierarchy_set_transpose0(h, ctypes.byref(M)))
        self._has_transpose0 = True

    def psolve(self, b):
        """Legacy interface: one iteration (multilevel.py:339-353)."""
        return self.solve(b, maxiter=1)

    def aspreconditioner(self, cycle="V"):
        """LinearOperator applying one cycle from x0 = 0 (multilevel.py:355-396), on NumPy arrays.  Its device
        form is ``solve(r, maxiter=1, cycle=cycle, tol=1e-12)`` on a CUDA tensor r: r and the result stay in device
        memory.  With one cycle the stop test cannot change the result, so ``tol=0`` gives the same tensor without
        the one norm read: that call only enqueues the cycle and returns."""
        shape = self.levels[0].A.shape
        dtype = self.levels[0].A.dtype

        def matvec(b):
            return self.solve(b, maxiter=1, cycle=cycle, tol=1e-12)

        M = LinearOperator(shape, matvec, dtype=dtype)
        M._amgb_solver, M._amgb_cycle = self, str(cycle).upper()     # lets pyamg_b200.krylov keep the solve resident
        return M

    def solve(self, b, x0=None, tol=1e-5, maxiter=100, cycle="V", accel=None, callback=None,
              residuals=None, cycles_per_level=1, return_info=False, out=None):
        """Execute multigrid cycling on the GPU (pyamg/multilevel.py:398-582; same arguments).

        ``out`` (extension, optional): a C-contiguous float64 array of n entries that receives the solution
        and is returned (reshaped like b) instead of a freshly allocated array -- with a page-locked buffer
        (``pyamg_b200.pinned_empty``) this removes the page-fault cost of a new 100+ MB result per call.

        CUDA tensors (extension): with ``b`` (and ``x0``, ``out``) ``torch.Tensor``s on ``cuda:<self.device>`` the
        solve reads and writes them in device memory -- no host copies -- and returns a float64 CUDA tensor of n
        entries (``out``, a contiguous float64 CUDA tensor, if given) with the iterate, info and residuals the host
        path computes on the same values.  Real dtypes are converted to float64 on the device; x0 is never written.
        The engine's work is ordered against ``torch.cuda.current_stream()``: it reads the inputs after the work
        enqueued there before the call, and later work there sees the result.  With ``tol=0`` and no
        ``residuals`` the call does not wait for the GPU; ``solve(r, maxiter=1, tol=1e-12)`` on a tensor is the
        device form of ``aspreconditioner()``.  ``accel`` may be 'cg', 'bicgstab', 'gmres', 'gmres_householder',
        'gmres_mgs', 'fgmres', 'cgnr', 'cgne', 'minimal_residual' or 'steepest_descent' (without a callback);
        ``callback`` (plain cycling) receives the device iterate after every cycle.

        Without a callback those ten ``accel`` names run GPU-resident, on host arrays and on tensors alike: the
        reference's function of that name (pyamg.krylov, criteria 'rr') with one cycle from zero as M, its maxiter
        default and clamp, its iterate, info, residual list and warnings.  'gmres_householder' is 'gmres'.  CGNR and
        CGNE keep A^H of the fine level on the device from their first call on, about the memory of A itself."""
        dev = _is_cuda(b) or _is_cuda(x0) or _is_cuda(out)
        if not dev:
            b = np.asarray(b)
        if out is not None and (accel is not None or callback is not None):
            raise ValueError("out= is supported for plain cycling only")
        if not dev:
            if out is not None and not (isinstance(out, np.ndarray) and out.dtype == np.float64
                                        and out.flags.c_contiguous and out.size == b.size):
                raise ValueError("out must be a C-contiguous float64 array with as many entries as b")
            if x0 is None:
                # the engine starts from zero on the device (AMGB_FLAG_X0_ZERO): the host buffer is output only
                x = out if out is not None else (np.empty_like(b, dtype=np.float64) if accel is None and callback is None
                                                 and not np.iscomplexobj(b) else np.zeros_like(b))
            else:
                x = np.array(x0)    # copy (:467)
                if out is not None:
                    np.copyto(out.reshape(x.shape), x)
                    x = out

        A = self.levels[0].A
        n = A.shape[0]
        cycle = self._check_cycle(cycle, accel)

        if accel is not None:
            spec = _resident(accel)
            resident = spec is not None and callback is None and n >= spec.min_n
            if dev and callback is not None:
                raise NotImplementedError("accel with a callback runs on host iterates: pass NumPy arrays")
            if dev and not resident:
                raise NotImplementedError(f"accel={accel!r} on this hierarchy runs a host solver, which needs NumPy "
                                          f"arrays; on CUDA tensors the accelerators are {_ACCEL_NAMES} (n >= 2 for "
                                          "the GMRES family and 'bicgstab')")
            if resident and (dev or not np.iscomplexobj(b)):
                # pyamg.krylov's function of that name (what the reference resolves the string to,
                # multilevel.py:495-499) with every long vector resident in HBM
                return self._solve_resident(accel, b, x0, tol, maxiter, cycle, residuals, return_info)
            if accel == "cg":
                accel = _cg_host           # same algorithm on the host (callback wants host iterates)
            elif isinstance(accel, str):
                # the reference looks the name up in pyamg.krylov first, then in scipy.sparse.linalg
                # (multilevel.py:495-499); its host solvers are used when the reference is importable, with the GPU
                # cycle as M (one host <-> device round trip per application)
                try:
                    from pyamg import krylov as ref_krylov
                except ImportError:
                    ref_krylov = None
                if ref_krylov is not None and hasattr(ref_krylov, accel):
                    accel = getattr(ref_krylov, accel)
                elif hasattr(sla, accel):
                    accel = getattr(sla, accel)
                else:
                    raise NotImplementedError(f"accel='{accel}': GPU-resident accelerators are {_ACCEL_NAMES}; "
                                              "other names need pyamg.krylov or scipy.sparse.linalg to provide a "
                                              "host solver of that name")
            M = self.aspreconditioner(cycle=cycle)
            try:  # PyAMG style interface which has a residuals parameter (multilevel.py:503-508)
                x, info = accel(A, b, x0=x0, tol=tol, maxiter=maxiter, M=M, callback=callback,
                                residuals=residuals)
                if return_info:
                    return x, info
                return x
            except TypeError:
                # scipy.sparse.linalg style interface (multilevel.py:509-535)
                if residuals is not None:
                    residuals[:] = [np.linalg.norm(b - A @ x)]

                    def callback_wrapper(xk):
                        if np.isscalar(xk):
                            residuals.append(xk)
                        else:
                            residuals.append(np.linalg.norm(b - A @ xk))
                        if callback is not None:
                            callback(xk)
                else:
                    callback_wrapper = callback
                x, info = accel(A, b, x0=x0, maxiter=maxiter, M=M, callback=callback_wrapper,
                                rtol=tol, atol=0)
                if return_info:
                    return x, info
                return x

        if dev:
            if maxiter < 1:
                raise ValueError("maxiter must be at least 1")
            bh, xh, flags = self._device_vectors(b, x0, out)
        else:
            if np.iscomplexobj(b) or np.iscomplexobj(x):
                raise NotImplementedError("complex systems are outside the fp64 hot path")
            if b.size != n or x.size != n:
                raise ValueError("b / x0 have invalid dimensions")
            if maxiter < 1:
                raise ValueError("maxiter must be at least 1")
            bh = np.ascontiguousarray(np.ravel(b), dtype=np.float64)        # :551-554
            xh = np.ascontiguousarray(np.ravel(x), dtype=np.float64)
            flags = E.FLAG_X0_ZERO if x0 is None else 0       # x0 = 0: no host->device copy of the guess

        L = E.lib()
        h = self.handle
        cyc = E.CYCLES[cycle]
        info = ctypes.c_int32(0)
        nres = ctypes.c_int32(0)

        if callback is None:
            # device operands, no residual list and tol = 0: the call only enqueues the cycles (no host synchronisation)
            res = np.empty(maxiter + 1, dtype=np.float64) if residuals is not None or not dev else None
            E.check(L.amgb_solve_ex(h, _ptr(bh), _ptr(xh), float(tol), int(maxiter), cyc, int(cycles_per_level), flags,
                                    None if res is None else E.f64p(res), ctypes.byref(nres), ctypes.byref(info)))
            if residuals is not None:
                residuals[:] = list(res[:nres.value])
            status = info.value
        else:
            # callback(x) wants the iterate after every cycle: one engine call per cycle from x (zero for x0=None);
            # the stop test scales with NumPy's ||b||
            if flags & E.FLAG_X0_ZERO:
                xh[:] = 0.0
                flags &= ~E.FLAG_X0_ZERO
            res = np.empty(2, dtype=np.float64)
            it = 0
            normb = np.linalg.norm(bh.cpu().numpy() if dev else bh)
            if normb == 0.0:
                normb = 1.0
            while True:
                E.check(L.amgb_solve_ex(h, _ptr(bh), _ptr(xh), 0.0, 1, cyc, int(cycles_per_level), flags,
                                        E.f64p(res), ctypes.byref(nres), ctypes.byref(info)))
                if it == 0 and residuals is not None:
                    residuals[:] = [res[0]]
                it += 1
                if residuals is not None:
                    residuals.append(res[1])
                callback(xh)
                if res[1] < tol * normb:
                    status = 0
                    break
                if it == maxiter:
                    status = it
                    break

        # b and x are ravelled before cycling (multilevel.py:553-554): (n,) out, even for (n,1) in
        xout = xh if dev else xh.ravel()
        if return_info:
            return xout, status
        return xout

    def _blocks(self, B, X0):
        """solve_many's B and X0 with their shapes checked, and whether they are CUDA tensors: NumPy arrays as
        given, or contiguous float64 tensors on this hierarchy's device (_device_operand)."""
        dev = _is_cuda(B) or _is_cuda(X0)
        if dev:
            B = self._device_operand(B, "B")
        else:
            B = np.asarray(B)
        n = self.levels[0].A.shape[0]
        if B.ndim != 2:
            raise ValueError("B must be a 2-D (n, k) array")
        if B.shape[0] != n or B.shape[1] < 1:
            raise ValueError("B has invalid dimensions")
        if X0 is not None:
            X0 = self._device_operand(X0, "X0") if dev else np.asarray(X0)
            if tuple(X0.shape) != tuple(B.shape):
                raise ValueError("X0 must have the shape of B")
        return B, X0, dev

    def solve_many(self, B, X0=None, tol=1e-5, maxiter=100, cycle="V", residuals=None, cycles_per_level=1,
                   return_info=False, accel=None):
        """Cycle k right-hand sides at once: column j of the result is ``solve(B[:, j], x0=X0[:, j], ...)``.

        B is an (n, k) array, X0 None (zeros) or of the same shape (copied, never modified).  Up to eight
        columns share each pass over the hierarchy, so the operator bytes a cycle streams are paid once per
        group instead of once per column.  Every column has its own ||b||, stop test and info; a column that
        converges keeps that cycle's iterate while the others go on.  Returns X, a C-contiguous float64 (n, k)
        array, or (X, info) with info an int array of length k.  If ``residuals`` is a list it is set to k
        lists, list j being what ``solve`` records for column j.  The batched cycle covers the smoothers none,
        Jacobi, Gauss-Seidel / SOR, block Jacobi, block Gauss-Seidel (the smoothed-aggregation default) and
        Chebyshev / Richardson, the normal-equation smoothers (``jacobi_ne``, ``gauss_seidel_ne``,
        ``gauss_seidel_nr``) and overlapping Schwarz (``schwarz``, ``strength_based_schwarz``), with a dense or a
        relaxation coarse solver of those kinds.  Hierarchies with another smoother (indexed Jacobi, CF / FC
        Jacobi, CF / FC block Jacobi), Schwarz subdomains too large for a batched group's shared memory (more than
        400 rows when k >= 5, 800 when k is 3 or 4, 1600 when k = 2), and AMLI cycles are solved column by column
        through ``solve``.

        ``accel='cg'``, ``'bicgstab'``, ``'gmres'``, ``'gmres_householder'``, ``'gmres_mgs'``, ``'fgmres'``,
        ``'cgnr'``, ``'cgne'``, ``'minimal_residual'`` or ``'steepest_descent'`` runs the GPU-resident Krylov method of
        ``solve(..., accel=accel)`` on all columns together (preconditioner = the batched cycle); column j, its
        info and its residual list are what ``solve(B[:, j], x0=X0[:, j], tol=tol, maxiter=maxiter, cycle=cycle,
        accel=accel)`` returns, and ``cycles_per_level`` is ignored, as ``solve`` ignores it.  GMRES keeps
        ``max_inner + 1`` Householder reflectors (or, for ``'gmres_mgs'``, Krylov basis vectors) per column on the
        device (``max_inner = min(maxiter, n)``, or ``min(n, 40)`` for ``maxiter=None``); when even two columns'
        vectors do not fit, the columns run one by one.  Any other ``accel`` runs column by column through
        ``solve``.  With ``accel`` each distinct warning is raised once per call, not once per column.

        CUDA tensors (extension): with B (and X0) ``torch.Tensor``s on ``cuda:<self.device>`` the blocks are read
        and X written in device memory, as ``solve`` does with tensors; X is an (n, k) float64 CUDA tensor, info
        and residuals are as above.  Plain cycling and the ten ``accel`` values above are supported; column by
        column solves go through ``solve`` on the tensor columns."""
        B, X0, dev = self._blocks(B, X0)
        if accel is None and maxiter < 1:
            raise ValueError("maxiter must be at least 1")
        if not dev and (np.iscomplexobj(B) or (X0 is not None and np.iscomplexobj(X0))):
            raise NotImplementedError("complex systems are outside the fp64 hot path")
        cycle = str(cycle).upper()
        if cycle not in E.CYCLES:
            raise TypeError(f"Unrecognized cycle type ({cycle})")
        k = B.shape[1]
        if accel is not None:
            done = self._solve_many_resident(B, X0, dev, tol, maxiter, cycle, residuals, return_info, accel)
            if done is not None:
                return done
        elif k > 1:
            Bh = B if dev else np.ascontiguousarray(B, dtype=np.float64)
            X = _new_block(B, X0, dev)
            # device blocks, no residual list and tol = 0: the call only enqueues the cycles
            res = np.empty((maxiter + 1, k), dtype=np.float64) if residuals is not None or not dev else None
            nres = np.zeros(k, dtype=np.int32)
            info = np.zeros(k, dtype=np.int32)
            flags = (E.FLAG_X0_ZERO if X0 is None else 0) | (self._device_io() if dev else 0)
            rc = E.lib().amgb_solve_many(self.handle, k, _ptr(Bh), _ptr(X), float(tol), int(maxiter),
                                         E.CYCLES[cycle], int(cycles_per_level),
                                         flags, None if res is None else E.f64p(res), E.i32p(nres),
                                         E.i32p(info))
            if rc != E.ENOTIMPL:
                E.check(rc)
                if residuals is not None:
                    residuals[:] = [list(res[:nres[j], j]) for j in range(k)]
                return (X, info.astype(int)) if return_info else X
        # k = 1, or a case the batched engine does not cover: column by column; every distinct warning of the k
        # solves is raised once
        spec = _resident(accel)
        X = _new_block(B, None, dev)
        info = np.zeros(k, dtype=int)
        lists = []
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            for j in range(k):
                rj = [] if residuals is not None else None
                xj, info[j] = self.solve(B[:, j], x0=None if X0 is None else X0[:, j], tol=tol, maxiter=maxiter,
                                         cycle=cycle, accel=accel if spec is None else spec.name, residuals=rj,
                                         cycles_per_level=cycles_per_level, return_info=True)
                X[:, j] = xj if dev else np.ravel(xj)
                lists.append(rj)
        seen = set()
        for w in caught:
            key = (w.category, str(w.message))
            if key not in seen:
                seen.add(key)
                warn(w.message)
        if residuals is not None:
            residuals[:] = lists
        return (X, info) if return_info else X

    def _solve_many_resident(self, B, X0, dev, tol, maxiter, cycle, residuals, return_info, accel):
        """solve_many(accel=accel) with the batched form of an accelerator of _ACCELS on all columns, with what
        solve warns raised once per call; None when the batched engine does not take the case."""
        spec = _resident(accel)
        n, k = B.shape
        if spec is None or k == 1 or cycle == "AMLI" or n < spec.min_n:
            return None
        its, rows, clamp = spec.iterations(maxiter, n)
        if spec.transpose:
            self._transpose0()
        Bh = B if dev else np.ascontiguousarray(B, dtype=np.float64)
        X = _new_block(B, X0, dev, zero=True)
        # the GMRES entries always take a residual buffer, of `rows` rows
        res = np.empty((rows, k), dtype=np.float64) if residuals is not None or spec.entry == "gmres" else None
        nres, info, reason = (np.zeros(k, dtype=np.int32) for _ in range(3))
        flags = (E.FLAG_X0_ZERO if X0 is None else 0) | (self._device_io() if dev else 0)
        rc = spec.call(self.handle, k, _ptr(Bh), _ptr(X), tol, its, E.CYCLES[cycle], flags, res, nres, info, reason)
        if rc == E.ENOTIMPL:
            return None
        E.check(rc)
        if spec.name == "cg" and not self.symmetric_smoothing:
            warn(_SPD_WARNING)
        if clamp is not None:
            warn(clamp)
        for text in spec.stop_warnings(info, reason):
            warn(text)
        if residuals is not None:
            residuals[:] = [list(res[:nres[j], j]) for j in range(k)]
        info = info.astype(int)
        return (X, info) if return_info else X
