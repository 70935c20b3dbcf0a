"""Hierarchies built under different AMGB_* launch settings, or on different devices, used side by side.

Every hierarchy keeps the settings it was created under, so solves on two of them -- interleaved on one thread,
concurrent on two threads, or on two GPUs -- compute bit for bit what each computes alone."""
import os
import threading

import numpy as np
import pytest

from conftest import golden_path
from pyamg_b200 import _engine as E
from pyamg_b200.hierarchy_io import load_hierarchy

pytestmark = pytest.mark.gpu

NAME = "cfg3_rs_mcgs_poisson3d"
# the defaults, and another tile geometry on every level with fp64 values and plain stream-ordered launches
SETTINGS = [{}, {"AMGB_TILE_CFG": "4", "AMGB_TILE_MIN_NNZ": "0", "AMGB_NO_VALUE_CODES": "1", "AMGB_NO_PDL": "1"}]


def _build(monkeypatch, env, device=0):
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        ml, ex = load_hierarchy(golden_path(NAME), device=device)
        ml.upload()                                  # the settings are read here
    return ml, ex["b"]


def _solves(ml, b):
    """Iterates (as bits) and residual lists of a few solves on ml."""
    out = []
    for cycle, accel, maxiter in (("V", None, 4), ("W", None, 3), ("V", "cg", 4)):
        res = []
        x = ml.solve(b, tol=0, maxiter=maxiter, cycle=cycle, accel=accel, residuals=res)
        out.append((np.ascontiguousarray(x).view(np.uint64).copy(), [float(r).hex() for r in res]))
    return out


def _alone(monkeypatch, env, device=0):
    ml, b = _build(monkeypatch, env, device)
    ref = _solves(ml, b)
    ml._invalidate()
    return ref


def _same(got, ref):
    assert len(got) == len(ref)
    for (x, res), (x_ref, res_ref) in zip(got, ref):
        assert np.array_equal(x, x_ref)
        assert res == res_ref


def test_interleaved_hierarchies(monkeypatch):
    refs = [_alone(monkeypatch, env) for env in SETTINGS]
    built = [_build(monkeypatch, env) for env in SETTINGS]
    for _ in range(2):
        for i, (ml, b) in enumerate(built):
            _same(_solves(ml, b), refs[i])


@pytest.mark.skipif(os.environ.get("AMGB_TEST_EMU") == "1", reason="the kernel emulator's built-ins are process globals")
def test_concurrent_hierarchies(monkeypatch):
    refs = [_alone(monkeypatch, env) for env in SETTINGS]
    built = [_build(monkeypatch, env) for env in SETTINGS]
    for _ in range(3):
        got, errors = [None] * len(built), []
        start = threading.Barrier(len(built))

        def run(i):
            try:
                start.wait()
                got[i] = _solves(*built[i])
            except BaseException as exc:     # noqa: BLE001 - reported on the main thread
                errors.append(exc)

        threads = [threading.Thread(target=run, args=(i,)) for i in range(len(built))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        for i in range(len(built)):
            _same(got[i], refs[i])


def test_two_devices(monkeypatch):
    if E.lib().amgb_device_count() < 2:
        pytest.skip("needs two CUDA devices")
    env = SETTINGS[1]                                # tile kernels that opt in to large shared memory on each device
    refs = [_alone(monkeypatch, env, device) for device in (0, 1)]
    built = [_build(monkeypatch, env, device) for device in (0, 1)]
    for i, (ml, b) in enumerate(built):
        _same(_solves(ml, b), refs[i])
