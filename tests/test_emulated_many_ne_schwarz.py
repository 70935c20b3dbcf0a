"""solve_many with the normal-equation smoothers and overlapping Schwarz on the kernel emulator (tests/emu): a bounded
subset of tests/test_gpu_many_ne_schwarz.py -- the four golden hierarchies at k = 3 and k = 11, their tolerance stop,
one accelerator per kind of smoother, the host-setup sweeps, the relaxation coarse solvers and the oversized Schwarz
subdomains -- also with bulk copies completing only at the wait (AMGB_EMU_TMA=lazy), run in a child process with
AMGB_TEST_EMU=1 as tests/test_emulated_many_widening.py does."""
import platform
import shutil

import pytest

from test_emulated_engine import _run

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64" or shutil.which("g++") is None,
                                reason="the fiber emulator needs x86-64 and g++")

SUBSET = ("(columns_match and (3 or 11)) or tolerance_stop "
          "or (accelerated and (cfg13 and gmres or cfg14 and minimal_residual or cfg15 and cg)) "
          "or host_setup_every_sweep or relaxation_coarse_solvers or oversized_schwarz")


@pytest.mark.parametrize("extra", [{}, {"AMGB_EMU_TMA": "lazy"}])
def test_solve_many_ne_schwarz_subset_on_the_emulator(extra):
    out = _run(extra, SUBSET, files=("tests/test_gpu_many_ne_schwarz.py",), timeout=1800)
    assert "failed" not in out
