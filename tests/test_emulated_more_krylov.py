"""solve / solve_many(accel='cgnr' | 'cgne' | 'minimal_residual' | 'steepest_descent') on the kernel emulator
(tests/emu): a bounded subset of tests/test_gpu_more_krylov.py -- the batched columns against per-column solves on a
symmetric (cfg2) and a nonsymmetric (cfg9's advection operator) hierarchy, k = 3 and 8, host blocks, plus the
transpose's refresh after change_solve_matrix -- run in a child process with AMGB_TEST_EMU=1, as
tests/test_emulated_engine.py does.  (The device-block variants need CUDA tensors, which the emulator has not.)"""
import platform
import shutil

import pytest

from test_emulated_engine import _run

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64" or shutil.which("g++") is None,
                                reason="the fiber emulator needs x86-64 and g++")

# one child process per width, each within _run's time limit
SUBSETS = {"k3": "(many_columns_equal_solve and host and k3) or transpose_follows",
           "k8": "many_columns_equal_solve and host and k8"}


@pytest.mark.parametrize("width", sorted(SUBSETS))
def test_more_krylov_subset_on_the_emulator(width):
    out = _run({}, SUBSETS[width], files=("tests/test_gpu_more_krylov.py",))
    assert "failed" not in out
