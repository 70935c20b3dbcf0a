"""solve_many with block Gauss-Seidel, polynomial smoothers and relaxation coarse solvers on the kernel emulator
(tests/emu): a bounded subset of tests/test_gpu_many_widening.py -- cfg7, cfg10, cfg11 and two adopted hierarchies,
k = 3 and k = 8, one Krylov pair, the forced kernel paths of cfg10 and the device-byte accounting -- also with bulk
copies completing only at the wait (AMGB_EMU_TMA=lazy), run in a child process with AMGB_TEST_EMU=1 as
tests/test_emulated_many.py does."""
import platform
import shutil

import pytest

from test_emulated_engine import _run

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64" or shutil.which("g++") is None,
                                reason="the fiber emulator needs x86-64 and g++")

SUBSET = ("(columns_match and (cfg7 or cfg10 or cfg11 or sa_default or sa_energy_chebyshev)) "
          "or (w_and_f and (cfg10 or cfg11)) or (widths_and_groups and (3 or 8)) "
          "or (tolerance_stop and (cfg7 or cfg11)) or (krylov and cfg10) or batched_launches "
          "or (kernel_paths and cfg10) or device_bytes")


@pytest.mark.parametrize("extra", [{}, {"AMGB_EMU_TMA": "lazy"}])
def test_solve_many_widening_subset_on_the_emulator(extra):
    out = _run(extra, SUBSET, files=("tests/test_gpu_many_widening.py",))
    assert "failed" not in out
