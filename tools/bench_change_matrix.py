#!/usr/bin/env python
"""bench_change_matrix.py -- MultilevelSolver.change_solve_matrix on a resident hierarchy against a full re-upload.

    python tools/bench_change_matrix.py [--workloads cfg3,cfg2,cfg5] [--reps 3] [--out FILE]

For each workload (bench.build_hierarchy at the bench's default sizes: cfg3 = Poisson 256^3 + RS + multi-colour
symmetric Gauss-Seidel, cfg2 = Poisson 2000^2 + SA + Jacobi, cfg5 = elasticity 300^2 BSR + SA + block Jacobi) two
changes of the fine matrix are timed, alternating with the matrix the hierarchy was built on:

  same_pattern : c * A (c = 2 and back to 1): the values change, the pattern does not (level 0 refreshed in place)
  pattern      : A plus one symmetric off-diagonal block pair and its weight on the diagonal (level 0 rebuilt)

each as the new path (change_solve_matrix, which replaces level 0 on the device) and as the old one (the same level and
smoother update followed by ml._invalidate(), so the first solve uploads the whole hierarchy again).  Per repetition
and variant: wall time of the change plus the first solve(b, maxiter=1) ending in a device synchronise; the change
alone; rebuild_smoother alone (host work both variants share); the path taken and the hierarchy's device bytes.
The two variants alternate, and their iterates must agree bit for bit.  The card's name and power limit are read in
the same run.  Prints one JSON line (and writes it to --out).  Needs an NVIDIA GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definitions and sizes)
from tools.bench_device_io import gpu_info  # noqa: E402


def pattern_change(A):
    """A plus one symmetric off-diagonal pair (first and last block row) with its weight moved onto the diagonal."""
    bs = A.blocksize[0] if sp.isspmatrix_bsr(A) else 1
    n = A.shape[0]
    i, j = 0, n - bs
    r = [i, j, i, j]
    c = [j, i, i, j]
    E = sp.csr_matrix(([-1e-3, -1e-3, 1e-3, 1e-3], (r, c)), shape=A.shape)
    B = (sp.csr_matrix(A) + E).tocsr()
    return sp.bsr_matrix(B, blocksize=A.blocksize) if bs > 1 else B


def measure(name, reps):
    import torch
    from pyamg_b200 import _engine as E
    from pyamg_b200.relaxation import smoothing
    bench.WORKLOAD["name"] = name
    g = bench.DEFAULT_GRID[name]
    ml = bench.build_hierarchy((g,) * 3)
    t0 = time.perf_counter()
    ml.upload()
    upload_s = time.perf_counter() - t0
    A1 = ml.levels[0].A
    n = A1.shape[0]
    b = np.random.default_rng(bench.SEED).random(n)
    ml.solve(b, maxiter=1, tol=1e-12)
    changes = {"same_pattern": 2.0 * A1, "pattern": pattern_change(A1)}

    def sync():
        torch.cuda.synchronize()

    def run(A, old):
        sync()
        t0 = time.perf_counter()
        if old:                               # what change_solve_matrix did before it kept the hierarchy resident
            ml.levels[0].A = A
            smoothing.rebuild_smoother(ml.levels[0])
            ml._invalidate()
            path = 0
        else:
            ml.change_solve_matrix(A)
            path = ml._last_replace_path
        sync()
        t1 = time.perf_counter()
        x = ml.solve(b, maxiter=1, tol=1e-12)
        sync()
        t2 = time.perf_counter()
        return {"total_s": t2 - t0, "change_s": t1 - t0, "first_solve_s": t2 - t1, "path": path,
                "device_bytes": int(E.lib().amgb_hierarchy_device_bytes(ml.handle))}, x

    out = {"n": int(n), "nnz0": int(sp.csr_matrix(A1).nnz), "levels": len(ml.levels), "full_upload_s": round(upload_s, 3)}
    for tag, A2 in changes.items():
        ml.levels[0].A = A2
        t0 = time.perf_counter()
        smoothing.rebuild_smoother(ml.levels[0])
        rebuild_s = time.perf_counter() - t0
        ml.change_solve_matrix(A1)            # back to the built matrix, resident
        ml.solve(b, maxiter=1, tol=1e-12)
        rows = {"new": [], "old": []}
        same = True
        for _ in range(reps):
            for variant in ("new", "old"):
                r, x = run(A2, variant == "old")
                rows[variant].append((r, x))
                run(A1, variant == "old")     # and back, so that every timed change is a change
            same = same and bool(np.array_equal(rows["new"][-1][1], rows["old"][-1][1]))
        res = {"rebuild_smoother_s": round(rebuild_s, 3), "bitwise_equal": same}
        for variant, rr in rows.items():
            med = {k: float(np.median([r[k] for r, _ in rr])) for k in ("total_s", "change_s", "first_solve_s")}
            res[variant] = {k: round(v, 4) for k, v in med.items()}
            res[variant]["path"] = rr[-1][0]["path"]
            res[variant]["device_bytes"] = rr[-1][0]["device_bytes"]
        res["speedup_total"] = round(res["old"]["total_s"] / res["new"]["total_s"], 2)
        out[tag] = res
        bench.log(f"[{name}] {tag}: {res}")
    del ml
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2,cfg5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_change_matrix.py needs an NVIDIA GPU")
    card, power = gpu_info()
    res = {"gpu": card, "power_limit": power}
    for name in args.workloads.split(","):
        res[name] = measure(name, args.reps)
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
