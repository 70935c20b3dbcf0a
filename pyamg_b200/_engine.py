"""ctypes binding of the C ABI in include/pyamg_b200.h (libpyamg_b200.so).

There is deliberately NO fallback: if the CUDA library is missing or no CUDA device is visible,
every entry point raises.  (The reference-side binding a pyamg maintainer would add is this file's
shape: see INTEGRATION.md.)
"""
import ctypes
import os

import numpy as np

from . import build as _build

c_i32p = ctypes.POINTER(ctypes.c_int32)
c_f64p = ctypes.POINTER(ctypes.c_double)

OK, EINVAL, ECUDA, ENOTIMPL, ESTATE = 0, -1, -2, -3, -4
SM_NONE, SM_JACOBI, SM_GAUSS_SEIDEL, SM_BLOCK_JACOBI = 0, 1, 2, 3
SM_POLYNOMIAL, SM_JACOBI_INDEXED, SM_CF_JACOBI, SM_FC_JACOBI, SM_BLOCK_GAUSS_SEIDEL = 4, 5, 6, 7, 8
SM_CF_BLOCK_JACOBI, SM_FC_BLOCK_JACOBI = 9, 10
SM_JACOBI_NE, SM_GAUSS_SEIDEL_NE, SM_GAUSS_SEIDEL_NR, SM_SCHWARZ = 11, 12, 13, 14
SWEEPS = {"forward": 0, "backward": 1, "symmetric": 2}
CYCLES = {"V": 0, "W": 1, "F": 2, "AMLI": 3}
FLAG_X0_ZERO = 1
FLAG_FLEXIBLE = 2
FLAG_DEVICE_IO = 4
FLAG_MGS = 8                    # amgb_solve_gmres / amgb_solve_many_gmres: modified Gram-Schmidt GMRES
FLAG_REORTH = 16                # with FLAG_MGS: gmres_mgs(reorth=True)
# amgb_solve_krylov / amgb_solve_many_krylov: the method argument (AMGB_KRYLOV_*) and the reason for info = -1
KRYLOV = {"cgnr": 0, "cgne": 1, "minimal_residual": 2, "steepest_descent": 3}
REASON_INDEFINITE_MATRIX, REASON_INDEFINITE_PRECONDITIONER, REASON_SINGULAR_PRECONDITIONER = 1, 2, 3
CUDA_STREAM_LEGACY = 1          # cudaStreamLegacy: the handle of the legacy default stream (torch's cuda_stream 0)


class Matrix(ctypes.Structure):
    _fields_ = [("n_rows", ctypes.c_int32), ("n_cols", ctypes.c_int32),
                ("block_r", ctypes.c_int32), ("block_c", ctypes.c_int32),
                ("nnz_blocks", ctypes.c_int64),
                ("indptr", c_i32p), ("indices", c_i32p), ("data", c_f64p)]


class Smoother(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int32), ("iterations", ctypes.c_int32),
                ("sweep", ctypes.c_int32), ("blocksize", ctypes.c_int32),
                ("omega", ctypes.c_double),
                ("indices", c_i32p), ("n_indices", ctypes.c_int64),
                ("Dinv", c_f64p),
                ("indices2", c_i32p), ("n_indices2", ctypes.c_int64),
                ("f_iterations", ctypes.c_int32), ("c_iterations", ctypes.c_int32),
                ("coefficients", c_f64p), ("n_coefficients", ctypes.c_int32), ("reserved_", ctypes.c_int32)]


class EngineError(RuntimeError):
    pass


_lib = None

# every symbol include/pyamg_b200.h declares (tests check the .so exports all of them)
SYMBOLS = [
    "amgb_last_error", "amgb_version", "amgb_device_count",
    "amgb_hierarchy_create", "amgb_hierarchy_destroy", "amgb_hierarchy_add_level",
    "amgb_hierarchy_set_coarse_pinv", "amgb_hierarchy_set_coarse_relaxation", "amgb_hierarchy_finalize",
    "amgb_hierarchy_set_io_stream", "amgb_solve", "amgb_solve_ex", "amgb_solve_cg",
    "amgb_solve_gmres", "amgb_solve_bicgstab",
    "amgb_solve_device", "amgb_solve_many", "amgb_solve_many_device", "amgb_solve_many_cg", "amgb_solve_many_bicgstab",
    "amgb_solve_many_gmres", "amgb_solve_krylov", "amgb_solve_many_krylov", "amgb_hierarchy_set_transpose0",
    "amgb_hierarchy_replace_level0",
    "amgb_hierarchy_num_levels", "amgb_hierarchy_device_bytes",
    "amgb_hierarchy_last_launches", "amgb_profile_cycle", "amgb_host_alloc", "amgb_host_free",
    "amgb_operator_create", "amgb_operator_destroy", "amgb_operator_apply",
    "amgb_host_jacobi", "amgb_host_gauss_seidel", "amgb_host_sor_gauss_seidel",
    "amgb_host_gauss_seidel_indexed",
    "amgb_host_bsr_jacobi", "amgb_host_block_jacobi", "amgb_host_matvec",
    "amgb_host_jacobi_indexed", "amgb_host_block_gauss_seidel", "amgb_host_relax",
    "amgb_host_csr_matmat", "amgb_free",
    "amgb_arnoldi_create", "amgb_arnoldi_run", "amgb_arnoldi_combine", "amgb_arnoldi_destroy",
    "amgb_dev_csr_spmv", "amgb_dev_csr_residual", "amgb_dev_csr_spmv_add", "amgb_dev_csr_jacobi",
    "amgb_dev_csr_gs_wave", "amgb_dev_partials_len", "amgb_dev_dense_matvec", "amgb_dev_fill",
    "amgb_dev_gather", "amgb_dev_reduce_len", "amgb_dev_dot", "amgb_dev_axpby", "amgb_dev_block_jacobi",
    "amgb_wave_schedule", "amgb_debug_build_tiles",
    "amgb_host_vertex_coloring_mis",
    "amgb_comm_create", "amgb_comm_connect", "amgb_comm_exchange", "amgb_comm_destroy",
]


def lib():
    """Load libpyamg_b200.so (building it in-tree when nvcc is around). Raises if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.build_extension()
    if not os.path.exists(path):
        raise EngineError("libpyamg_b200.so is missing: run `python -m pyamg_b200.build` "
                          "(there is no CPU fallback)")
    _lib = _bind(ctypes.CDLL(path))
    return _lib


def _bind(L):
    """Declare the C signatures of include/pyamg_b200.h on a loaded library object."""
    L.amgb_last_error.restype = ctypes.c_char_p
    L.amgb_hierarchy_device_bytes.restype = ctypes.c_int64
    L.amgb_hierarchy_last_launches.restype = ctypes.c_int64
    L.amgb_dev_partials_len.restype = ctypes.c_int64
    L.amgb_hierarchy_destroy.restype = None
    vp, i32, i64, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
    L.amgb_hierarchy_create.argtypes = [ctypes.c_int, ctypes.POINTER(vp)]
    L.amgb_hierarchy_destroy.argtypes = [vp]
    L.amgb_hierarchy_add_level.argtypes = [vp, ctypes.POINTER(Matrix), ctypes.POINTER(Matrix),
                                           ctypes.POINTER(Matrix), ctypes.POINTER(Smoother),
                                           ctypes.POINTER(Smoother)]
    L.amgb_hierarchy_set_coarse_pinv.argtypes = [vp, i32, c_f64p, i32]
    L.amgb_hierarchy_set_coarse_relaxation.argtypes = [vp, ctypes.POINTER(Smoother)]
    L.amgb_hierarchy_finalize.argtypes = [vp, vp]
    L.amgb_hierarchy_set_io_stream.argtypes = [vp, vp]
    L.amgb_solve.argtypes = [vp, vp, vp, f64, i32, i32, i32, c_f64p, c_i32p, c_i32p]
    L.amgb_solve_ex.argtypes = [vp, vp, vp, f64, i32, i32, i32, i32, c_f64p, c_i32p, c_i32p]
    L.amgb_solve_cg.argtypes = [vp, vp, vp, f64, i32, i32, i32, c_f64p, c_i32p, c_i32p]
    L.amgb_solve_bicgstab.argtypes = [vp, vp, vp, f64, i32, i32, i32, c_f64p, c_i32p, c_i32p]
    L.amgb_solve_gmres.argtypes = [vp, vp, vp, f64, i32, i32, i32, i32, c_f64p, i32, c_i32p, c_i32p]
    L.amgb_solve_device.argtypes = [vp, vp, vp, i32, i32, i32, vp]
    L.amgb_solve_many.argtypes = [vp, i32, vp, vp, f64, i32, i32, i32, i32, c_f64p, c_i32p, c_i32p]
    L.amgb_solve_many_device.argtypes = [vp, i32, vp, vp, i32, i32, i32, vp]
    L.amgb_solve_many_cg.argtypes = [vp, i32, vp, vp, f64, i32, i32, i32, c_f64p, c_i32p, c_i32p]
    L.amgb_solve_many_bicgstab.argtypes = [vp, i32, vp, vp, f64, i32, i32, i32, c_f64p, c_i32p, c_i32p]
    L.amgb_solve_many_gmres.argtypes = [vp, i32, vp, vp, f64, i32, i32, i32, i32, c_f64p, i32, c_i32p, c_i32p]
    L.amgb_solve_krylov.argtypes = [vp, i32, vp, vp, f64, i32, i32, i32, c_f64p, c_i32p, c_i32p, c_i32p]
    L.amgb_solve_many_krylov.argtypes = [vp, i32, i32, vp, vp, f64, i32, i32, i32, c_f64p, c_i32p, c_i32p, c_i32p]
    L.amgb_hierarchy_set_transpose0.argtypes = [vp, ctypes.POINTER(Matrix)]
    L.amgb_hierarchy_replace_level0.argtypes = [vp, ctypes.POINTER(Matrix), ctypes.POINTER(Smoother),
                                                ctypes.POINTER(Smoother), vp, c_i32p]
    L.amgb_hierarchy_num_levels.argtypes = [vp]
    L.amgb_hierarchy_device_bytes.argtypes = [vp]
    L.amgb_hierarchy_last_launches.argtypes = [vp]
    L.amgb_profile_cycle.argtypes = [vp, i32, c_f64p, i32, c_i32p]
    L.amgb_operator_create.argtypes = [ctypes.c_int, ctypes.POINTER(Matrix), ctypes.POINTER(ctypes.c_int64), i32,
                                       vp, ctypes.POINTER(vp)]
    L.amgb_operator_destroy.argtypes = [vp]
    L.amgb_operator_destroy.restype = None
    L.amgb_operator_apply.argtypes = [vp, i32, vp, vp, vp, vp, f64, vp, i32]
    L.amgb_host_alloc.argtypes = [ctypes.c_size_t, ctypes.POINTER(vp)]
    L.amgb_host_free.argtypes = [vp]
    ci = ctypes.c_int
    L.amgb_host_jacobi.argtypes = [c_i32p, ci, c_i32p, ci, c_f64p, ci, c_f64p, ci, c_f64p, ci,
                                   c_f64p, ci, i32, i32, i32, c_f64p, ci]
    L.amgb_host_gauss_seidel.argtypes = [c_i32p, ci, c_i32p, ci, c_f64p, ci, c_f64p, ci, c_f64p, ci,
                                         i32, i32, i32]
    L.amgb_host_sor_gauss_seidel.argtypes = [c_i32p, ci, c_i32p, ci, c_f64p, ci, c_f64p, ci, c_f64p, ci,
                                             i32, i32, i32, f64]
    L.amgb_host_gauss_seidel_indexed.argtypes = [c_i32p, ci, c_i32p, ci, c_f64p, ci, c_f64p, ci,
                                                 c_f64p, ci, c_i32p, ci, i32, i32, i32]
    L.amgb_host_bsr_jacobi.argtypes = [c_i32p, ci, c_i32p, ci, c_f64p, ci, c_f64p, ci, c_f64p, ci,
                                       c_f64p, ci, i32, i32, i32, i32, c_f64p, ci]
    L.amgb_host_block_jacobi.argtypes = [c_i32p, ci, c_i32p, ci, c_f64p, ci, c_f64p, ci, c_f64p, ci,
                                         c_f64p, ci, c_f64p, ci, i32, i32, i32, c_f64p, ci, i32]
    L.amgb_host_matvec.argtypes = [ctypes.POINTER(Matrix), c_f64p, c_f64p]
    L.amgb_host_jacobi_indexed.argtypes = [c_i32p, ci, c_i32p, ci, c_f64p, ci, c_f64p, ci, c_f64p, ci,
                                           c_i32p, ci, c_f64p, ci]
    L.amgb_host_block_gauss_seidel.argtypes = [c_i32p, ci, c_i32p, ci, c_f64p, ci, c_f64p, ci, c_f64p, ci,
                                               c_f64p, ci, i32, i32, i32, i32]
    L.amgb_host_csr_matmat.argtypes = [ctypes.POINTER(Matrix), ctypes.POINTER(Matrix), ctypes.POINTER(c_i32p),
                                       ctypes.POINTER(c_i32p), ctypes.POINTER(c_f64p), ctypes.POINTER(ctypes.c_int64)]
    L.amgb_arnoldi_create.argtypes = [ctypes.c_int, ctypes.POINTER(Matrix), c_f64p, i32, ctypes.POINTER(vp)]
    L.amgb_arnoldi_run.argtypes = [vp, c_f64p, f64, c_f64p, c_i32p]
    L.amgb_arnoldi_combine.argtypes = [vp, c_f64p, i32]
    L.amgb_arnoldi_destroy.argtypes = [vp]
    L.amgb_arnoldi_destroy.restype = None
    L.amgb_free.argtypes = [vp]
    L.amgb_free.restype = None
    L.amgb_host_relax.argtypes = [ctypes.POINTER(Matrix), ctypes.POINTER(Smoother), c_f64p, c_f64p]
    L.amgb_dev_csr_spmv.argtypes = [i32, vp, vp, vp, vp, vp, ci, vp]
    L.amgb_dev_csr_residual.argtypes = [i32, vp, vp, vp, vp, vp, vp, vp, vp, ci, vp]
    L.amgb_dev_csr_spmv_add.argtypes = [i32, vp, vp, vp, vp, vp, ci, vp]
    L.amgb_dev_csr_jacobi.argtypes = [i32, vp, vp, vp, vp, vp, vp, vp, f64, ci, vp]
    L.amgb_dev_csr_gs_wave.argtypes = [i32, i32, vp, vp, vp, vp, vp, vp, f64, ci, vp]
    L.amgb_dev_partials_len.argtypes = [i32, ci]
    L.amgb_dev_dense_matvec.argtypes = [i32, i32, vp, vp, vp, vp]
    L.amgb_dev_fill.argtypes = [vp, i64, f64, vp]
    L.amgb_dev_gather.argtypes = [vp, vp, vp, i64, vp]
    L.amgb_dev_reduce_len.restype = ctypes.c_int64
    L.amgb_dev_reduce_len.argtypes = []
    L.amgb_dev_dot.argtypes = [vp, vp, i64, vp, vp, vp]
    L.amgb_dev_axpby.argtypes = [f64, vp, f64, vp, i64, vp]
    L.amgb_dev_block_jacobi.argtypes = [i32, i32, vp, vp, vp, vp, vp, vp, vp, f64, ci, vp]
    L.amgb_debug_build_tiles.argtypes = [i32, c_i32p, i32, ctypes.POINTER(ctypes.c_int64), i32, i32, i32, c_i32p,
                                         c_i32p, i32, c_i32p, c_i32p]
    L.amgb_wave_schedule.argtypes = [i32, c_i32p, c_i32p, c_i32p, i64, c_i32p, c_i32p]
    L.amgb_host_vertex_coloring_mis.argtypes = [i32, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p]
    L.amgb_comm_create.argtypes = [ci, ci, ci, i64, vp, ctypes.POINTER(vp), ctypes.c_char_p]
    L.amgb_comm_connect.argtypes = [vp, ctypes.c_char_p, ctypes.c_uint32]
    L.amgb_comm_exchange.argtypes = [vp, vp, i64, vp, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64), i64]
    L.amgb_comm_destroy.argtypes = [vp]
    L.amgb_comm_destroy.restype = None
    return L


def check(rc):
    """Map C error codes onto the exception types the reference raises for the same misuse."""
    if rc == OK:
        return
    msg = lib().amgb_last_error().decode("utf8", "replace")
    if rc == EINVAL:
        raise ValueError(msg)
    if rc == ENOTIMPL:
        raise NotImplementedError(msg)
    if rc == ESTATE:
        raise EngineError("engine state: " + msg)
    raise EngineError("CUDA: " + msg)


def require_gpu():
    if lib().amgb_device_count() < 1:
        raise EngineError("no CUDA device visible: pyamg_b200 has no CPU fallback")


def i32p(a):
    return a.ctypes.data_as(c_i32p)


def f64p(a):
    return a.ctypes.data_as(c_f64p)


def as_matrix(M, keep):
    """scipy csr/bsr (any object with .format/.indptr/.indices/.data) -> C `amgb_matrix`.

    Normalised arrays are appended to `keep` so they outlive the ctypes struct.
    """
    fmt = getattr(M, "format", None)
    if fmt not in ("csr", "bsr"):
        M = M.tocsr()
        fmt = "csr"
    if M.dtype != np.float64:
        if np.issubdtype(M.dtype, np.complexfloating):
            raise NotImplementedError("complex operators are outside the fp64 hot path")
        M = M.astype(np.float64)
    indptr = np.ascontiguousarray(M.indptr, dtype=np.int32)
    indices = np.ascontiguousarray(M.indices, dtype=np.int32)
    data = np.ascontiguousarray(M.data, dtype=np.float64)
    R, C = (M.blocksize if fmt == "bsr" else (1, 1))
    keep += [indptr, indices, data]
    return Matrix(int(M.shape[0]), int(M.shape[1]), int(R), int(C), int(len(indices)),
                  i32p(indptr), i32p(indices), f64p(data.reshape(-1)))


def pinned_empty(n, dtype=np.float64):
    """Page-locked host array (cudaHostAlloc) for the e2e path; freed when garbage-collected."""
    dtype = np.dtype(dtype)
    p = ctypes.c_void_p()
    check(lib().amgb_host_alloc(ctypes.c_size_t(int(n) * dtype.itemsize), ctypes.byref(p)))
    buf = (ctypes.c_char * (int(n) * dtype.itemsize)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dtype, count=int(n))
    _PINNED[id(arr)] = (p, arr)   # keep alive; released by free_pinned
    return arr


_PINNED = {}


def free_pinned(arr):
    ent = _PINNED.pop(id(arr), None)
    if ent is not None:
        lib().amgb_host_free(ent[0])


def csr_matmat(A, B):
    """C = A @ B on the GPU with SciPy's csr_matmat results bit for bit (amgb_host_csr_matmat): the Galerkin
    product of the setup phase (pyamg/classical/classical.py:201).  Returns a scipy csr_array."""
    from scipy import sparse
    if A.shape[1] != B.shape[0]:
        raise ValueError("dimension mismatch")
    require_gpu()
    keep = []
    MA, MB = as_matrix(sparse.csr_array(A), keep), as_matrix(sparse.csr_array(B), keep)
    Cp, Cj, Cx, nnz = c_i32p(), c_i32p(), c_f64p(), ctypes.c_int64(0)
    check(lib().amgb_host_csr_matmat(MA, MB, ctypes.byref(Cp), ctypes.byref(Cj), ctypes.byref(Cx), ctypes.byref(nnz)))
    try:
        n, m = A.shape[0], nnz.value
        indptr = np.ctypeslib.as_array(Cp, shape=(n + 1,)).copy()
        indices = np.ctypeslib.as_array(Cj, shape=(max(m, 1),))[:m].copy()
        data = np.ctypeslib.as_array(Cx, shape=(max(m, 1),))[:m].copy()
    finally:
        for p in (Cp, Cj, Cx):
            lib().amgb_free(ctypes.cast(p, ctypes.c_void_p))
    return sparse.csr_array((data, indices, indptr), shape=(A.shape[0], B.shape[1]))
