"""change_solve_matrix on a resident hierarchy (tests/test_gpu_change_matrix.py) on the kernel emulator (tests/emu):
the in-place refresh and the level-0 rebuild."""
import os
import platform
import shutil
import subprocess
import sys

import pytest

from conftest import ROOT

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64" or shutil.which("g++") is None,
                                reason="the fiber emulator needs x86-64 and g++")

# one case per mechanism, small enough for the emulator: a level-0 rebuild (path 2), the in-place refresh with the
# normal-equation slot maps (cfg13) and the Schwarz copy (cfg15), row-coded level-0 values, the one-level fallback
SUBSET = ("(test_pattern_change_rebuilds_level0 and cfg1 and True) or (test_scaled_matrix_refreshes_in_place and cfg13) "
          "or (test_every_level0_smoother_kind and cfg15) or test_one_level_hierarchy_falls_back "
          "or (test_every_level0_stream_format and cfg2 and ROW_MIN_NNZ and not NO_ROW and not GRAPH)")


def test_change_matrix_on_the_emulator():
    env = dict(os.environ, AMGB_TEST_EMU="1")
    cmd = [sys.executable, "-m", "pytest", "tests/test_gpu_change_matrix.py", "-m", "gpu", "-q", "-x",
           "-p", "no:cacheprovider", "-k", SUBSET]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
