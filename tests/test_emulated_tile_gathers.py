"""The batched tile-kernel gathers (tests/test_gpu_tile_gathers.py) on the kernel emulator (tests/emu), in the default,
reversed and shuffled thread orders and with bulk copies that complete only when waited for."""
import os
import platform
import shutil
import subprocess
import sys

import pytest

from conftest import ROOT

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64" or shutil.which("g++") is None,
                                reason="the fiber emulator needs x86-64 and g++")


@pytest.mark.parametrize("extra", [{}, {"AMGB_EMU_ORDER": "reverse"}, {"AMGB_EMU_ORDER": "random:20261017"},
                                   {"AMGB_EMU_TMA": "lazy", "AMGB_EMU_SMS": "1"}])
def test_tile_gathers_on_the_emulator(extra):
    env = dict(os.environ, AMGB_TEST_EMU="1", **extra)
    cmd = [sys.executable, "-m", "pytest", "tests/test_gpu_tile_gathers.py", "-m", "gpu", "-q", "-x",
           "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
