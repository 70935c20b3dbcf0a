#!/usr/bin/env python
"""bench_gmres_mgs.py -- modified Gram-Schmidt GMRES resident on the GPU (solve / solve_many(accel='gmres_mgs')).

    python tools/bench_gmres_mgs.py [--grid 256] [--maxiters 20,40] [--reps 3] [--out FILE]

On the headline hierarchy (bench.build_hierarchy: Poisson grid^3, RS, multi-colour symmetric Gauss-Seidel), with the
same seeded right-hand side and tol = 0 (so every call runs exactly `maxiter` inner iterations):

  (a) resident gmres_mgs against the reference's host pyamg.krylov.gmres_mgs with the GPU cycle as M (one host <->
      device round trip per application), when the reference is importable from oracle/_ref/site; one call, at the
      smallest maxiter only (the host method takes minutes at 256^3)
  (b) resident gmres_mgs against resident Householder GMRES (accel='gmres'), ms per inner iteration
  (c) solve_many(accel='gmres_mgs') at k = 4 and 8 against k single calls, column-iterations per second

Per-call wall time: host clock around the call, which ends in a device synchronise (the residual read), after one
warm-up call; (b) alternates the two methods per repetition.  Outputs are checked against each other: (a) and (b)
relative difference of the iterates, (c) every batched column equal to its single solve bit for bit.  The card's
name and power limit are read in the same run.  Prints one JSON line (and writes it to --out).  Needs an NVIDIA GPU:
without one it exits with an error.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definitions and sizes)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power = (out[0].split(",") + ["?"])[:2] if out else ("?", "?")
    return name.strip(), power.strip()


def relerr(a, b):
    return float(np.linalg.norm(np.ravel(a) - np.ravel(b)) / max(np.linalg.norm(np.ravel(b)), 1e-300))


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--maxiters", default="20,40")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--widths", default="4,8")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    maxiters = [int(m) for m in args.maxiters.split(",")]
    widths = [int(k) for k in args.widths.split(",")]
    from pyamg_b200 import _engine as E
    if E.lib().amgb_device_count() < 1:
        sys.exit("bench_gmres_mgs: no CUDA device")
    warnings.simplefilter("ignore")
    card, power = gpu_info()
    bench.WORKLOAD["name"] = "cfg3"
    ml = bench.build_hierarchy((args.grid,) * 3)
    ml.upload()
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(bench.SEED)
    b = rng.random(n)
    out = {"card": card, "power_limit": power, "workload": f"poisson({args.grid}^3) RS multi-colour symmetric GS",
           "n": n, "tol": 0.0}

    def solve(accel, m):
        return ml.solve(b, tol=0.0, maxiter=m, accel=accel, return_info=True)

    # (b) resident MGS vs resident Householder
    for m in maxiters:
        for accel in ("gmres_mgs", "gmres"):
            solve(accel, m)                                           # warm-up: buffers of this shape
        t = {"gmres_mgs": [], "gmres": []}
        x = {}
        for _ in range(args.reps):
            for accel in ("gmres_mgs", "gmres"):
                dt, (xa, info) = timed(lambda: solve(accel, m))
                t[accel].append(dt)
                x[accel] = (xa, info)
        its = {a: (x[a][1] if x[a][1] > 0 else m) for a in x}
        out[f"maxiter{m}"] = {
            "mgs_ms_per_iter": 1e3 * min(t["gmres_mgs"]) / its["gmres_mgs"],
            "householder_ms_per_iter": 1e3 * min(t["gmres"]) / its["gmres"],
            "mgs_over_householder_time": min(t["gmres_mgs"]) / min(t["gmres"]),
            "info": {a: int(x[a][1]) for a in x},
            "relerr_mgs_vs_householder": relerr(x["gmres_mgs"][0], x["gmres"][0]),
        }

    # (a) the reference's host gmres_mgs with the GPU cycle as M
    site = os.path.join(ROOT, "oracle", "_ref", "site")
    if os.path.isdir(site):
        sys.path.insert(0, site)
    try:
        from pyamg.krylov import gmres_mgs as ref_gmres_mgs
    except ImportError:
        ref_gmres_mgs = None
    m = min(maxiters)
    if ref_gmres_mgs is not None:
        M = ml.aspreconditioner()
        dt_ref, (x_ref, info_ref) = timed(lambda: ref_gmres_mgs(ml.levels[0].A, b, tol=0.0, maxiter=m, M=M))
        dt_res, (x_res, info_res) = timed(lambda: solve("gmres_mgs", m))
        out["host_reference"] = {"maxiter": m, "host_ms_per_iter": 1e3 * dt_ref / m,
                                 "resident_ms_per_iter": 1e3 * dt_res / m, "speedup": dt_ref / dt_res,
                                 "info": [int(info_ref), int(info_res)], "relerr_vs_reference": relerr(x_res, x_ref)}
    else:
        out["host_reference"] = "not measured: the reference is not importable from oracle/_ref/site"

    # (c) solve_many at k columns against k single calls
    for k in widths:
        B = rng.random((n, k))
        ml.solve_many(B, tol=0.0, maxiter=m, accel="gmres_mgs")     # warm-up: the K-wide basis store
        t_many, t_single = [], []
        for _ in range(args.reps):
            dt, X = timed(lambda: ml.solve_many(B, tol=0.0, maxiter=m, accel="gmres_mgs"))
            t_many.append(dt)
            t0 = time.perf_counter()
            xs = [ml.solve(B[:, j], tol=0.0, maxiter=m, accel="gmres_mgs") for j in range(k)]
            t_single.append(time.perf_counter() - t0)
        same = all(np.array_equal(X[:, j], xs[j]) for j in range(k))
        out[f"many_k{k}"] = {"maxiter": m, "batched_col_iters_per_s": k * m / min(t_many),
                             "single_col_iters_per_s": k * m / min(t_single),
                             "speedup": min(t_single) / min(t_many), "columns_equal_single_bitwise": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
