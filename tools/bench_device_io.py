#!/usr/bin/env python
"""bench_device_io.py -- MultilevelSolver.solve / solve_many on NumPy arrays against the same calls on CUDA tensors.

    python tools/bench_device_io.py [--workloads cfg3,cfg5] [--reps 20] [--out FILE]

For each workload (bench.build_hierarchy at the bench's default sizes: cfg3 = Poisson 256^3 + RS + multi-colour
symmetric Gauss-Seidel, the headline; cfg5 = elasticity 300^2 + SA + block Jacobi) the same seeded inputs go through
host arrays and through CUDA tensors (AMGB_FLAG_DEVICE_IO: no host copies of the vectors):

  (a) solve(b, maxiter=1, tol=1e-12)                  the preconditioner application aspreconditioner() makes
  (b) solve(b, tol=1e-8)
  (c) solve(b, accel='cg', tol=1e-8)
  (d) solve_many(B, accel='fgmres', tol=0, maxiter=20) with k = 8

Per-call wall time: host clock around `reps` calls (2 for (d)) ending in a device synchronise, after one warm-up call
of each; the host and device variants alternate per repetition, so both see the same machine state.  Every device
output is compared with the host output bit for bit.  The card's name and power limit are read in the same run.
Prints one JSON line (and writes it to --out).  Needs an NVIDIA GPU: without one it exits with an error.
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


def to_host(v):
    return v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)


def measure(name, reps):
    import torch
    bench.WORKLOAD["name"] = name
    g = bench.DEFAULT_GRID[name]
    ml = bench.build_hierarchy((g,) * 3)
    ml.upload()
    n = ml.levels[0].A.shape[0]
    rng = np.random.default_rng(bench.SEED)
    b = rng.random(n)
    B = rng.random((n, 8))
    bd = torch.from_numpy(b).cuda()
    Bd = torch.from_numpy(B).cuda()
    cases = {
        "a_precond": (lambda v: ml.solve(v, maxiter=1, tol=1e-12), b, bd, reps),
        "b_tol1e-8": (lambda v: ml.solve(v, tol=1e-8, return_info=True), b, bd, max(reps // 4, 2)),
        "c_cg_tol1e-8": (lambda v: ml.solve(v, accel="cg", tol=1e-8, return_info=True), b, bd, max(reps // 4, 2)),
        "d_many_fgmres_k8": (lambda v: ml.solve_many(v, accel="fgmres", tol=0, maxiter=20, return_info=True),
                             B, Bd, 2),
    }
    out = {"n": int(n)}
    for tag, (fn, host_in, dev_in, r) in cases.items():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            rh, rd = fn(host_in), fn(dev_in)                 # warm-up (and the outputs compared below)
            torch.cuda.synchronize()
            th = td = 0.0
            for _ in range(r):
                t0 = time.perf_counter()
                fn(host_in)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                fn(dev_in)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                th += t1 - t0
                td += t2 - t1
        xh, xd = (rh[0], rd[0]) if isinstance(rh, tuple) else (rh, rd)
        same = bool(np.array_equal(to_host(xh), to_host(xd)))
        if isinstance(rh, tuple):
            same = same and bool(np.array_equal(np.asarray(rh[1]), np.asarray(rd[1])))
        out[tag] = {"host_ms": round(1e3 * th / r, 3), "device_ms": round(1e3 * td / r, 3),
                    "saved_ms": round(1e3 * (th - td) / r, 3), "speedup": round(th / td, 3), "reps": r,
                    "bitwise_equal": same}
        if isinstance(rh, tuple):
            out[tag]["info"] = np.asarray(rh[1]).tolist()
        bench.log(f"[{name}] {tag}: {out[tag]}")
    out["vector_MB"] = round(8 * n / 1e6, 1)
    del ml
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg5")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_device_io.py needs an NVIDIA GPU")
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
