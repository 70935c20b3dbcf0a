"""Batched x gathers of csr_tile_kernel (tile_kernels.cuh stage_gather): each lane reads the columns of its next
kTileBatch entries, issues their x loads back to back and only then sums the products, in stored order.  Rows of every
length modulo kTileBatch * G, diagonals duplicated across batch boundaries (the last one wins), zero diagonals and a
row longer than a tile, on G = 1, 2 and 4 lanes per row and with tiles on every launch, must give the oracle's
iterates."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from conftest import golden_path, relerr
from pyamg_b200.hierarchy_io import load_hierarchy

pytestmark = pytest.mark.gpu

TOL = 1e-12
_KNOBS = ("AMGB_TILE_G", "AMGB_TILE_MIN_NNZ", "AMGB_TILE_DENSE_CFG", "AMGB_NO_VALUE_CODES", "AMGB_NO_PAIR_CODES",
          "AMGB_NO_ZERO_START", "AMGB_NO_WAVE_RESID")


def _env(monkeypatch, env):
    for k in _KNOBS:
        if k in env:
            monkeypatch.setenv(k, env[k])
        else:
            monkeypatch.delenv(k, raising=False)


def _check(ml, b, cycle="V", accel=None):
    kw = {"accel": accel} if accel is not None else {}
    x = ml.solve(b, tol=0.0, maxiter=3, cycle=cycle, **kw)
    launches = ml.profile_cycle(cycle)
    ml._invalidate()
    cyc = oracle.Cycle(oracle.hierarchy_spec(ml), coarse_pinv=ml.coarse_solver.P)
    xo = cyc.solve(b, tol=0.0, maxiter=3, cycle=cycle, **kw)
    assert relerr(x, xo) < TOL
    return launches


def _ragged(A, rng):
    """A with extra entries so that row i holds 1 + (i mod 53) more (rows of every length modulo 4 G up to 60),
    a duplicated diagonal (stored apart, so that the two copies fall into different batches) on every 7th row, a
    zero diagonal on every 29th row and one row of 400 entries (longer than any tile)."""
    A = A.tocsr()
    n = A.shape[0]
    rows, cols, vals = [], [], []
    for i in range(n):
        s, e = A.indptr[i], A.indptr[i + 1]
        c, v = list(A.indices[s:e]), list(A.data[s:e])
        k = 400 if i == n // 3 else 1 + i % 53
        extra = rng.choice(n, size=min(k, n), replace=False)
        extra = extra[extra != i]
        c += list(extra)
        v += list(-1e-3 * rng.random(extra.size))
        if i % 7 == 0:
            c.append(i)
            v.append(50.0 + i % 5)
        if i % 29 == 0:
            v = [0.0 if cc == i else vv for cc, vv in zip(c, v)]
        rows += [i] * len(c)
        cols += c
        vals += v
    return _keep_order(rows, cols, vals, n)


def _keep_order(rows, cols, vals, n):
    """CSR with the entries of each row in the order given (duplicates kept, not summed)."""
    indptr = np.zeros(n + 1, dtype=np.int32)
    np.add.at(indptr, np.asarray(rows) + 1, 1)
    indptr = np.cumsum(indptr).astype(np.int32)
    return sp.csr_matrix((np.asarray(vals, dtype=float), np.asarray(cols, dtype=np.int32), indptr), shape=(n, n))


@pytest.mark.parametrize("G", ["1", "2", "4"])
@pytest.mark.parametrize("smoother", [("jacobi", {"omega": 0.7}), ("sor", {"omega": 1.3, "sweep": "symmetric"})])
def test_tile_gathers_ragged_rows(monkeypatch, G, smoother):
    """Level 0 of a 2-D Poisson RS hierarchy made ragged, under Jacobi and symmetric SOR."""
    from pyamg_b200.relaxation.smoothing import change_smoothers
    _env(monkeypatch, {"AMGB_TILE_G": G, "AMGB_TILE_MIN_NNZ": "0"})
    ml, ex = load_hierarchy(golden_path("cfg1_rs_gs_poisson2d"))
    ml.levels[0].A = _ragged(ml.levels[0].A, np.random.default_rng(11))
    change_smoothers(ml, smoother, smoother)
    _check(ml, ex["b"].ravel())


@pytest.mark.parametrize("G", ["2", "4"])
@pytest.mark.parametrize("cycle", ["V", "W", "F"])
@pytest.mark.parametrize("env", [{}, {"AMGB_NO_ZERO_START": "1", "AMGB_NO_WAVE_RESID": "1"},
                                 {"AMGB_NO_VALUE_CODES": "1"}])
def test_tile_gathers_multicolour_gauss_seidel(monkeypatch, G, cycle, env):
    """Multi-colour Gauss-Seidel waves, their last-wave residuals and zero-start copies on G lanes per row."""
    _env(monkeypatch, dict(env, AMGB_TILE_G=G, AMGB_TILE_MIN_NNZ="0"))
    ml, ex = load_hierarchy(golden_path("cfg3_rs_mcgs_poisson3d"))
    launches = _check(ml, ex["b"].ravel(), cycle=cycle)
    assert (launches[:, 1] == 4).any()


@pytest.mark.parametrize("accel", ["cg", "bicgstab"])
def test_tile_gathers_krylov(monkeypatch, accel):
    _env(monkeypatch, {"AMGB_TILE_G": "2", "AMGB_TILE_MIN_NNZ": "0"})
    ml, ex = load_hierarchy(golden_path("cfg3_rs_mcgs_poisson3d"))
    _check(ml, ex["b"].ravel(), accel=accel)
