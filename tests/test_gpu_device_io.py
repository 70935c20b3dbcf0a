"""solve / solve_many on CUDA tensors (AMGB_FLAG_DEVICE_IO): right-hand sides and iterates stay in device memory.

A device solve must compute exactly what the host solve computes on the same values -- iterate, info and residual
list, bit for bit -- since only the copies in and out differ.  The C-ABI tests (names with `c_abi`) also run on the
kernel emulator, where host memory announced as device allocations stands for device memory.
"""
import ctypes
import os
import warnings

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu
EMU = os.environ.get("AMGB_TEST_EMU") == "1"
ACCELS = ("cg", "bicgstab", "gmres", "fgmres")


def _torch_cuda():
    try:
        import torch
    except ImportError:
        return None
    return torch if torch.cuda.is_available() and not EMU else None


needs_cuda = pytest.mark.skipif(_torch_cuda() is None, reason="needs torch with a CUDA device")


def _cuda(a):
    return _torch_cuda().from_numpy(np.ascontiguousarray(a)).cuda()


def _quiet(fn, *args, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*args, **kw)


def _same_solve(ml, b, x0=None, **kw):
    """Device solve == host solve, bit for bit: iterate, info, residual list."""
    torch = _torch_cuda()
    rh, rd = [], []
    xh, ih = _quiet(ml.solve, b, x0=x0, residuals=rh, return_info=True, **kw)
    bd = _cuda(b)
    x0d = None if x0 is None else _cuda(x0)
    x0_before = None if x0d is None else x0d.clone()
    xd, idv = _quiet(ml.solve, bd, x0=x0d, residuals=rd, return_info=True, **kw)
    assert isinstance(xd, torch.Tensor) and xd.is_cuda and xd.dtype == torch.float64
    assert tuple(xd.shape) == xh.shape, kw
    assert np.array_equal(xd.cpu().numpy(), xh), kw
    assert idv == ih and rd == rh, kw
    if x0d is not None:
        assert torch.equal(x0d, x0_before)
    return xd


def _same_many(ml, B, X0=None, **kw):
    torch = _torch_cuda()
    rh, rd = [], []
    Xh, ih = _quiet(ml.solve_many, B, X0=X0, residuals=rh, return_info=True, **kw)
    X0d = None if X0 is None else _cuda(X0)
    X0_before = None if X0d is None else X0d.clone()
    Xd, idv = _quiet(ml.solve_many, _cuda(B), X0=X0d, residuals=rd, return_info=True, **kw)
    assert isinstance(Xd, torch.Tensor) and Xd.is_cuda and tuple(Xd.shape) == Xh.shape and Xd.is_contiguous()
    assert np.array_equal(Xd.cpu().numpy(), Xh), kw
    assert list(idv) == list(ih) and rd == rh, kw
    if X0d is not None:
        assert torch.equal(X0d, X0_before)


@needs_cuda
@pytest.mark.parametrize("name", GOLDEN)
def test_device_solve_equals_host_solve(name, load_golden):
    ml, ex = load_golden(name)
    b, x0 = ex["b"].ravel(), ex["x0"].ravel()
    cycles = ("V", "W", "F", "AMLI") if name.startswith("cfg3") else ("V", "W", "F")
    for cycle in cycles:
        for tol in (0.0, 1e-8):
            for guess in (None, x0):
                _same_solve(ml, b, x0=guess, tol=tol, maxiter=6, cycle=cycle)
    _same_solve(ml, b, x0=x0, tol=1e-8, maxiter=4, cycle="W", cycles_per_level=2)
    _same_solve(ml, b, tol=0, maxiter=3, cycle="F", cycles_per_level=2)
    for accel in ACCELS:
        _same_solve(ml, b, tol=1e-8, maxiter=10, accel=accel)
        _same_solve(ml, b, x0=x0, tol=1e-10, maxiter=8, accel=accel, cycle="W")
    if name.startswith("cfg3"):
        _same_solve(ml, b, x0=x0, tol=1e-8, maxiter=5, accel="fgmres", cycle="AMLI")


@needs_cuda
@pytest.mark.parametrize("k", [3, 8, 11])
@pytest.mark.parametrize("name", ["cfg2_sa_jacobi_poisson2d", "cfg3_rs_mcgs_poisson3d", "cfg5_sa_bjacobi_elasticity",
                                  "cfg9_air_fcjacobi_advection2d"])
def test_device_solve_many_equals_host(name, k, load_golden):
    """cfg9 (AIR: CF / FC Jacobi) is one of the hierarchies the batched engine leaves to per-column solves."""
    ml, ex = load_golden(name)
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(k)
    B = rng.standard_normal((n, k))
    B[:, 0] = ex["b"].ravel()
    X0 = rng.standard_normal((n, k))
    for X in (None, X0):
        _same_many(ml, B, X, tol=1e-8, maxiter=5)
        _same_many(ml, B, X, tol=0, maxiter=3, cycle="W")
        for accel in ACCELS:
            _same_many(ml, B, X, tol=1e-8, maxiter=6, accel=accel)


@needs_cuda
def test_device_solve_many_amli_and_fallback_accel(load_golden):
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    B = np.random.default_rng(4).standard_normal((n, 3))
    _same_many(ml, B, tol=1e-8, maxiter=4, cycle="AMLI")
    _same_many(ml, B, B.copy(), tol=1e-8, maxiter=4, cycle="AMLI", accel="fgmres")
    _same_many(ml, B[:, :1], tol=1e-8, maxiter=4)                     # k = 1: through solve


@needs_cuda
def test_inputs_and_outputs(load_golden):
    torch = _torch_cuda()
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    b = ex["b"].ravel()
    xh = ml.solve(b, tol=1e-8, maxiter=5)
    # (n, 1) input: the host path ravels
    assert np.array_equal(ml.solve(_cuda(b.reshape(n, 1)), tol=1e-8, maxiter=5).cpu().numpy(), xh)
    # float32 input: converted to float64 on the device, as the host path converts
    b32 = b.astype(np.float32)
    assert np.array_equal(ml.solve(_cuda(b32), tol=1e-8, maxiter=5).cpu().numpy(),
                          ml.solve(b32, tol=1e-8, maxiter=5))
    # out=
    out = torch.full((n,), 7.0, dtype=torch.float64, device="cuda")
    got = ml.solve(_cuda(b), tol=1e-8, maxiter=5, out=out)
    assert got.data_ptr() == out.data_ptr() and np.array_equal(out.cpu().numpy(), xh)
    with pytest.raises(ValueError):
        ml.solve(_cuda(b), out=torch.empty(n, dtype=torch.float32, device="cuda"))
    # column-major block ((k, n).T) and float32 blocks
    B = np.random.default_rng(2).standard_normal((n, 5))
    Xh = ml.solve_many(B, tol=1e-8, maxiter=4)
    Bt = _cuda(np.ascontiguousarray(B.T)).T
    assert not Bt.is_contiguous()
    assert np.array_equal(ml.solve_many(Bt, tol=1e-8, maxiter=4).cpu().numpy(), Xh)
    assert np.array_equal(ml.solve_many(_cuda(B.astype(np.float32)), tol=1e-8, maxiter=4).cpu().numpy(),
                          ml.solve_many(B.astype(np.float32), tol=1e-8, maxiter=4))
    # CPU tensors keep the host path and its return type
    x_cpu = ml.solve(torch.from_numpy(b), tol=1e-8, maxiter=5)
    assert isinstance(x_cpu, np.ndarray) and np.array_equal(x_cpu, xh)
    assert isinstance(ml.solve_many(torch.from_numpy(B), tol=1e-8, maxiter=4), np.ndarray)
    # pyamg_b200.krylov passes device b through
    from pyamg_b200 import krylov
    M = ml.aspreconditioner()
    for fn in (krylov.cg, krylov.gmres, krylov.fgmres, krylov.bicgstab):
        rh, rd = [], []
        x1, i1 = _quiet(fn, ml.levels[0].A, b, tol=1e-8, maxiter=6, M=M, residuals=rh)
        x2, i2 = _quiet(fn, ml.levels[0].A, _cuda(b), tol=1e-8, maxiter=6, M=M, residuals=rd)
        assert x2.is_cuda and np.array_equal(x2.cpu().numpy(), x1) and i1 == i2 and rh == rd
    # callback on plain cycling: the device iterate after every cycle, as on the host
    seen_h, seen_d = [], []
    xh2 = ml.solve(b, tol=1e-8, maxiter=4, callback=lambda x: seen_h.append(x.copy()))
    xd2 = ml.solve(_cuda(b), tol=1e-8, maxiter=4, callback=lambda x: seen_d.append(x.cpu().numpy()))
    assert np.array_equal(xd2.cpu().numpy(), xh2) and len(seen_h) == len(seen_d)
    assert all(np.array_equal(p, q) for p, q in zip(seen_h, seen_d))


@needs_cuda
def test_ordering_without_synchronisation(load_golden):
    """The engine's reads wait for the caller's stream, and the call returns before the GPU is done: b is written
    on a side stream behind a long sleep, and the solve (tol = 0, no residuals) must neither wait on the host nor
    read b early."""
    torch = _torch_cuda()
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    b = ex["b"].ravel()
    xh = ml.solve(b, tol=0, maxiter=2)
    bd = torch.zeros(b.size, dtype=torch.float64, device="cuda")
    ml.solve(bd, tol=0, maxiter=2)                       # warm-up: upload, graph capture
    torch.cuda.synchronize()
    src = _cuda(b)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                   # on the order of 0.1 s
        bd.copy_(src)
        x = ml.solve(bd, tol=0, maxiter=2)
        busy = not side.query()
    assert busy
    torch.cuda.synchronize()
    assert np.array_equal(x.cpu().numpy(), xh)


@needs_cuda
def test_no_large_host_device_copies(load_golden, tmp_path):
    import json
    torch = _torch_cuda()
    from torch.profiler import ProfilerActivity, profile
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    n = ml.levels[0].A.shape[0]
    b = _cuda(ex["b"].ravel())
    B = _cuda(np.random.default_rng(1).standard_normal((n, 4)))
    calls = (lambda: ml.solve(b, tol=1e-8, maxiter=4), lambda: ml.solve(b, tol=1e-8, maxiter=6, accel="gmres"),
             lambda: ml.solve_many(B, tol=1e-8, maxiter=6, accel="cg"))
    for fn in calls:
        fn()                                             # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in calls:
            fn()
        torch.cuda.synchronize()
    trace = str(tmp_path / "trace.json")
    prof.export_chrome_trace(trace)
    events = json.load(open(trace))["traceEvents"]
    copies = [(e["name"], e.get("args", {}).get("bytes", 0)) for e in events
              if e.get("cat") == "gpu_memcpy" and ("HtoD" in e["name"] or "DtoH" in e["name"])]
    assert copies, "the trace lists no host <-> device copies at all (the stop test's scalars are expected)"
    assert any(e.get("cat") == "kernel" for e in events)
    assert not [c for c in copies if c[1] >= 8 * n], copies
    # and no more launches than the host path's
    host = ex["b"].ravel()
    for dev_call, host_call in ((lambda: ml.solve(b, tol=1e-8, maxiter=4), lambda: ml.solve(host, tol=1e-8, maxiter=4)),
                                (lambda: ml.solve(b, tol=1e-8, maxiter=6, accel="gmres"),
                                 lambda: ml.solve(host, tol=1e-8, maxiter=6, accel="gmres"))):
        host_call()
        lh = ml.last_launches()
        dev_call()
        assert ml.last_launches() <= lh


@needs_cuda
def test_validation(load_golden):
    torch = _torch_cuda()
    ml, ex = load_golden("cfg2_sa_jacobi_poisson2d")
    n = ml.levels[0].A.shape[0]
    b = _cuda(ex["b"].ravel())
    with pytest.raises(NotImplementedError):
        ml.solve(b.to(torch.complex128))
    with pytest.raises(ValueError):
        ml.solve(b[:-1])
    with pytest.raises(ValueError):
        ml.solve(b, x0=np.zeros(n))                      # a host x0 with a device b
    with pytest.raises(NotImplementedError):
        ml.solve(b, accel="cr")
    with pytest.raises(NotImplementedError):
        ml.solve(b, accel="cg", callback=lambda x: None)
    with pytest.raises(ValueError):
        ml.solve_many(b.reshape(n, 1).repeat(1, 3), X0=torch.zeros((n, 2), dtype=torch.float64, device="cuda"))
    with pytest.raises(NotImplementedError):
        ml.solve_many(b.reshape(n, 1).repeat(1, 3).to(torch.complex128))
    with pytest.raises(NotImplementedError):
        ml.solve_many(b.reshape(n, 1).repeat(1, 3), accel="cr")
    if torch.cuda.device_count() < 2:
        pytest.skip("wrong-device check needs a second GPU")
    with pytest.raises(ValueError):
        ml.solve(b.to("cuda:1"))


# ---------------------------------------------------------------- the C entries (also on the emulator)
class _DeviceBuffers:
    """Device copies of host arrays for the C entries: CUDA tensors on a GPU; on the emulator host copies announced
    as device allocations."""

    def __init__(self):
        from pyamg_b200 import _engine as E
        self.L = E.lib()
        self.keep = []

    def __call__(self, a):
        a = np.array(a, dtype=np.float64, order="C")
        if EMU:
            self.L.amgb_emu_register_allocation(ctypes.c_void_p(a.ctypes.data), ctypes.c_size_t(max(a.nbytes, 1)))
            self.keep.append(a)
            return a
        t = _torch_cuda().from_numpy(a).cuda()
        self.keep.append(t)
        return t

    @staticmethod
    def ptr(d):
        return d.ctypes.data if isinstance(d, np.ndarray) else d.data_ptr()

    @staticmethod
    def host(d):
        if isinstance(d, np.ndarray):
            return d.copy()
        _torch_cuda().cuda.synchronize()
        return d.cpu().numpy()

    def close(self):
        if EMU:
            for a in self.keep:
                self.L.amgb_emu_unregister_allocation(ctypes.c_void_p(a.ctypes.data))
        self.keep = []


def _entry_calls(E, L, h, n, k):
    """(name, call(b_ptr, x_ptr, flags, res, nres, info), vector shape, residual slots) for the eight entries."""
    V = E.CYCLES["V"]
    return [
        ("solve_ex", lambda b, x, f, r, nr, inf: L.amgb_solve_ex(h, b, x, 1e-8, 5, V, 1, f, E.f64p(r),
                                                                 E.i32p(nr), E.i32p(inf)), (n,), 6),
        ("cg", lambda b, x, f, r, nr, inf: L.amgb_solve_cg(h, b, x, 1e-8, 5, V, f, E.f64p(r), E.i32p(nr),
                                                           E.i32p(inf)), (n,), 6),
        ("bicgstab", lambda b, x, f, r, nr, inf: L.amgb_solve_bicgstab(h, b, x, 1e-8, 5, V, f, E.f64p(r),
                                                                       E.i32p(nr), E.i32p(inf)), (n,), 6),
        ("gmres", lambda b, x, f, r, nr, inf: L.amgb_solve_gmres(h, b, x, 1e-8, 0, 5, V, f | E.FLAG_FLEXIBLE,
                                                                 E.f64p(r), 8, E.i32p(nr), E.i32p(inf)), (n,), 8),
        ("many", lambda b, x, f, r, nr, inf: L.amgb_solve_many(h, k, b, x, 1e-8, 5, V, 1, f, E.f64p(r),
                                                               E.i32p(nr), E.i32p(inf)), (n, k), 6),
        ("many_cg", lambda b, x, f, r, nr, inf: L.amgb_solve_many_cg(h, k, b, x, 1e-8, 5, V, f, E.f64p(r),
                                                                     E.i32p(nr), E.i32p(inf)), (n, k), 6),
        ("many_bicgstab", lambda b, x, f, r, nr, inf: L.amgb_solve_many_bicgstab(h, k, b, x, 1e-8, 5, V, f,
                                                                                 E.f64p(r), E.i32p(nr),
                                                                                 E.i32p(inf)), (n, k), 6),
        ("many_gmres", lambda b, x, f, r, nr, inf: L.amgb_solve_many_gmres(h, k, b, x, 1e-8, 0, 5, V, f, E.f64p(r),
                                                                           8, E.i32p(nr), E.i32p(inf)), (n, k), 8),
    ]


@pytest.mark.parametrize("name", ["cfg1_rs_gs_poisson2d", "cfg3_rs_mcgs_poisson3d"])
def test_c_abi_device_io_equals_host_io(name, load_golden):
    """Every entry with AMGB_FLAG_DEVICE_IO on device buffers == the same entry on host arrays, bit for bit; x0 is
    read from x unless AMGB_FLAG_X0_ZERO.  cfg3's level 0 is permuted (gathers straight from the caller's memory)."""
    from pyamg_b200 import _engine as E
    L = E.lib()
    ml, ex = load_golden(name)
    h = ml.handle
    n, k = ml.levels[0].A.shape[0], 3
    E.check(L.amgb_hierarchy_set_io_stream(h, None))     # the buffers are ready before each call (synchronised)
    rng = np.random.default_rng(7)
    dev = _DeviceBuffers()
    try:
        for tag, call, shape, slots in _entry_calls(E, L, h, n, k):
            b = rng.standard_normal(shape)
            x0 = rng.standard_normal(shape)
            cols = shape[1] if len(shape) > 1 else 1
            for flags in (0, E.FLAG_X0_ZERO):
                out = []
                for io in (0, E.FLAG_DEVICE_IO):
                    r = np.zeros(slots * cols)
                    nr, inf = np.zeros(cols, dtype=np.int32), np.zeros(cols, dtype=np.int32)
                    if io:
                        bd, xd = dev(b), dev(x0)
                        if not EMU:
                            _torch_cuda().cuda.synchronize()
                        E.check(call(dev.ptr(bd), dev.ptr(xd), flags | io, r, nr, inf))
                        x = dev.host(xd)
                        assert np.array_equal(dev.host(bd), b), tag
                    else:
                        x = x0.copy()
                        E.check(call(b.ctypes.data, x.ctypes.data, flags, r, nr, inf))
                    out.append((x, r, nr, inf))
                (xh, rh, nh, ih), (xd, rd, nd, idv) = out
                assert np.array_equal(xh, xd), (tag, flags)
                assert np.array_equal(rh, rd) and np.array_equal(nh, nd) and np.array_equal(ih, idv), (tag, flags)
    finally:
        dev.close()


def test_c_abi_device_io_rejects_host_pointers(load_golden):
    from pyamg_b200 import _engine as E
    L = E.lib()
    ml, ex = load_golden("cfg1_rs_gs_poisson2d")
    h = ml.handle
    n, k = ml.levels[0].A.shape[0], 3
    E.check(L.amgb_hierarchy_set_io_stream(h, None))
    dev = _DeviceBuffers()
    try:
        for tag, call, shape, slots in _entry_calls(E, L, h, n, k):
            cols = shape[1] if len(shape) > 1 else 1
            b, x = np.ones(shape), np.full(shape, 3.0)
            bd, xd = dev(b), dev(x)
            for bp, xp in ((b.ctypes.data, x.ctypes.data), (dev.ptr(bd), x.ctypes.data),
                           (b.ctypes.data, dev.ptr(xd))):
                r = np.zeros(slots * cols)
                nr, inf = np.zeros(cols, dtype=np.int32), np.zeros(cols, dtype=np.int32)
                assert call(bp, xp, E.FLAG_DEVICE_IO, r, nr, inf) == E.EINVAL, tag
                assert "device memory" in L.amgb_last_error().decode(), tag
            assert np.array_equal(x, np.full(shape, 3.0)), tag            # nothing was written
        assert np.array_equal(dev.host(xd), np.full(shape, 3.0))
    finally:
        dev.close()


def test_c_abi_no_host_wait_without_residuals(load_golden):
    """tol = 0 and no residual list: info and n_residuals come back without reading the device."""
    from pyamg_b200 import _engine as E
    L = E.lib()
    ml, ex = load_golden("cfg3_rs_mcgs_poisson3d")
    h = ml.handle
    n = ml.levels[0].A.shape[0]
    E.check(L.amgb_hierarchy_set_io_stream(h, None))
    b = ex["b"].ravel()
    xh = np.zeros(n)
    E.check(L.amgb_solve_ex(h, b.ctypes.data, xh.ctypes.data, 0.0, 3, 0, 1, E.FLAG_X0_ZERO, None, None, None))
    dev = _DeviceBuffers()
    try:
        bd, xd = dev(b), dev(np.zeros(n))
        if not EMU:
            _torch_cuda().cuda.synchronize()
        nr, inf = ctypes.c_int32(-5), ctypes.c_int32(-5)
        E.check(L.amgb_solve_ex(h, dev.ptr(bd), dev.ptr(xd), 0.0, 3, 0, 1, E.FLAG_X0_ZERO | E.FLAG_DEVICE_IO, None,
                                ctypes.byref(nr), ctypes.byref(inf)))
        assert nr.value == 4 and inf.value == 3
        assert np.array_equal(dev.host(xd), xh)
        B = np.column_stack([b, -b, 2 * b])
        Xh = np.zeros((n, 3))
        E.check(L.amgb_solve_many(h, 3, np.ascontiguousarray(B).ctypes.data, Xh.ctypes.data, 0.0, 2, 0, 1,
                                  E.FLAG_X0_ZERO, None, None, None))
        Bd, Xd = dev(B), dev(np.zeros((n, 3)))
        if not EMU:
            _torch_cuda().cuda.synchronize()
        nres, info = np.zeros(3, dtype=np.int32), np.zeros(3, dtype=np.int32)
        E.check(L.amgb_solve_many(h, 3, dev.ptr(Bd), dev.ptr(Xd), 0.0, 2, 0, 1, E.FLAG_X0_ZERO | E.FLAG_DEVICE_IO,
                                  None, E.i32p(nres), E.i32p(info)))
        assert list(nres) == [3, 3, 3] and list(info) == [2, 2, 2]
        assert np.array_equal(dev.host(Xd), Xh)
    finally:
        dev.close()
