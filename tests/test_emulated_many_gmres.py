"""solve_many(accel='gmres' | 'fgmres') on the kernel emulator (tests/emu): a bounded subset of
tests/test_gpu_many_gmres.py -- cfg1, cfg2 and cfg5 with k = 3 and k = 8 (padding, both group widths, block Jacobi),
restarts through the C ABI and validation, also with bulk copies completing only at the wait (AMGB_EMU_TMA=lazy) and
every operator on the tile kernels -- run in a child process with AMGB_TEST_EMU=1, as tests/test_emulated_engine.py
does."""
import platform
import shutil

import pytest

from test_emulated_engine import _run

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64" or shutil.which("g++") is None,
                                reason="the fiber emulator needs x86-64 and g++")

SUBSET = ("(stop_at_different and (cfg1 or cfg2 or cfg5)) or (widths_and_groups and (-3- or -8-)) "
          "or (restarts and cfg1) or validation")


@pytest.mark.parametrize("extra", [{}, {"AMGB_EMU_TMA": "lazy", "AMGB_TILE_MIN_NNZ": "0"}])
def test_solve_many_gmres_subset_on_the_emulator(extra):
    out = _run(extra, SUBSET, files=("tests/test_gpu_many_gmres.py",))
    assert "failed" not in out
