"""AMGB_FLAG_DEVICE_IO on the kernel emulator (tests/emu): the C-ABI subset of tests/test_gpu_device_io.py -- every
entry on device buffers against the same entry on host arrays, the pointer check, and the call without a host wait
-- run in a child process with AMGB_TEST_EMU=1, as tests/test_emulated_engine.py does.  Host memory announced as
device allocations stands for device memory there."""
import platform
import shutil

import pytest

from test_emulated_engine import _run

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64" or shutil.which("g++") is None,
                                reason="the fiber emulator needs x86-64 and g++")


def test_device_io_c_abi_subset_on_the_emulator():
    out = _run({}, "c_abi", files=("tests/test_gpu_device_io.py",))
    assert "failed" not in out
