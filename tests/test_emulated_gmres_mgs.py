"""solve / solve_many(accel='gmres_mgs') on the kernel emulator (tests/emu): a bounded subset of
tests/test_gpu_gmres_mgs.py -- the reference goldens on two configurations, the batched columns against per-column
solves at k = 3 and 8 (host blocks), restarts and reorth through the C entries, the reorth pass on an exhausted
Krylov space and the flag validation -- run in a child process with AMGB_TEST_EMU=1, as tests/test_emulated_engine.py
does.  (The device-block variants need CUDA tensors, which the emulator has not.)"""
import platform
import shutil

import pytest

from test_emulated_engine import _run

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64" or shutil.which("g++") is None,
                                reason="the fiber emulator needs x86-64 and g++")

# one child process per subset, each within _run's time limit
SUBSETS = {"golden": "solve_matches_golden and (cfg1_ or cfg9_)",
           "k3": "(many_columns_equal_solve and host and k3 and cfg2) or restarts_and_reorth or reorth_pass "
                 "or flag_validation",
           "k8": "many_columns_equal_solve and host and k8 and cfg2"}


@pytest.mark.parametrize("subset", sorted(SUBSETS))
def test_gmres_mgs_subset_on_the_emulator(subset):
    out = _run({}, SUBSETS[subset], files=("tests/test_gpu_gmres_mgs.py",))
    assert "failed" not in out
