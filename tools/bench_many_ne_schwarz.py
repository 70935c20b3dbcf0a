#!/usr/bin/env python
"""bench_many_ne_schwarz.py -- throughput of MultilevelSolver.solve_many on hierarchies smoothed by the
normal-equation smoothers and by overlapping Schwarz, against single-vector cycles.

    python tools/bench_many_ne_schwarz.py [--workloads gsnr,jacobi_ne,schwarz] [--steps 10] [--warmup 3]
                                          [--gmres-maxiter 20] [--grid N]

Workloads: this repository's host setup, smoothed_aggregation_solver(poisson((700, 700))) (490 000 unknowns; the
host setup takes well under a minute per workload), np.random.seed(bench.SEED), with the smoothers installed by
pyamg_b200.relaxation.smoothing.change_smoothers:
    gsnr       symmetric gauss_seidel_nr pre and post (Kaczmarz column sweeps, conflict waves of A^T)
    jacobi_ne  jacobi_ne pre and post
    schwarz    symmetric schwarz pre and post (default subdomains: each row's sparsity pattern)

For each workload and k in {1, 2, 4, 8}: k columns of B and X resident in HBM, `steps` V-cycles each followed by the
per-column residual norm, timed with CUDA events after `warmup` cycles (k = 1 amgb_solve_device, k > 1
amgb_solve_many_device); batched cycles/s, column-cycles/s, its ratio to k = 1, and the largest absolute per-column
difference between the batched iterate and k = 1 runs of the same columns after 2 cycles (it must be 0).  For gsnr
also GMRES: k calls of solve(b_j, accel='gmres', tol=0, maxiter=ITS) against one solve_many(B, accel='gmres', ...)
on host blocks, host wall clock around each call; column-iterations/s, ratio to k = 1, speed-up over the k single
calls, largest difference.  Prints one JSON line with the card's name and power limit (a read-only nvidia-smi query).
Needs an NVIDIA GPU: without one the script exits with an error, there is no CPU timing.
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

TOOLS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, TOOLS)

import bench_many as BM  # noqa: E402  (device-block cycling, card query)
from bench_many import bench  # noqa: E402

KS = BM.KS
DEFAULT_GRID = 700
SMOOTHERS = {"gsnr": ("gauss_seidel_nr", {"sweep": "symmetric"}),
             "jacobi_ne": ("jacobi_ne", {}),
             "schwarz": ("schwarz", {"sweep": "symmetric"})}


def build(name, grid, stream=None):
    from pyamg_b200.aggregation import smoothed_aggregation_solver
    from pyamg_b200.gallery import poisson
    from pyamg_b200.relaxation.smoothing import change_smoothers
    if name not in SMOOTHERS:
        sys.exit(f"bench_many_ne_schwarz.py: unknown workload {name!r}")
    np.random.seed(bench.SEED)
    t0 = time.time()
    ml = smoothed_aggregation_solver(poisson((grid, grid)), stream=stream)
    change_smoothers(ml, SMOOTHERS[name], SMOOTHERS[name])
    bench.log(f"[{name}] setup {time.time() - t0:.1f}s, levels {[lv.A.shape[0] for lv in ml.levels]}, "
              f"op-cx {ml.operator_complexity():.3f}")
    ml.upload()
    return ml


def measure_cycles(name, ml, args):
    import torch
    from pyamg_b200 import _engine as E
    n = ml.levels[0].A.shape[0]
    dev = torch.device("cuda")
    Bfull = torch.from_numpy(np.random.default_rng(bench.SEED).random((n, max(KS)))).to(dev)
    out, base = {}, None
    for k in KS:
        B = Bfull[:, :k].contiguous()
        X = torch.zeros((n, k), dtype=torch.float64, device=dev)
        norms = torch.zeros((args.steps + args.warmup + 1) * k, dtype=torch.float64, device=dev)
        BM.run_cycles(E, ml, k, B, X, args.warmup, norms)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        BM.run_cycles(E, ml, k, B, X, args.steps, norms)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        cps = 1e3 / ms
        if k == 1:
            base = cps
        X2 = torch.zeros((n, k), dtype=torch.float64, device=dev)       # parity: 2 cycles from zero
        BM.run_cycles(E, ml, k, B, X2, 2, norms)
        launches = ml.last_launches()
        diff = 0.0
        for j in range(k):
            xj = torch.zeros(n, dtype=torch.float64, device=dev)
            BM.run_cycles(E, ml, 1, B[:, j].contiguous(), xj, 2, norms)
            torch.cuda.synchronize()
            diff = max(diff, float((X2[:, j] - xj).abs().max()))
        out[str(k)] = {"cycles_per_s": round(cps, 2), "column_cycles_per_s": round(k * cps, 2),
                       "ratio_vs_k1": round(k * cps / base, 3), "ms_per_cycle": round(ms, 3),
                       "launches_per_2_cycles": launches, "max_col_abs_diff_vs_k1": diff}
        bench.log(f"[{name}] k={k}: {out[str(k)]}")
    return out


def measure_gmres(name, ml, args):
    n = ml.levels[0].A.shape[0]
    its = args.gmres_maxiter
    Bfull = np.random.default_rng(bench.SEED).random((n, max(KS)))
    kw = dict(accel="gmres", tol=0, maxiter=its)
    out, base = {}, None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for k in KS:
            B = np.ascontiguousarray(Bfull[:, :k])
            ml.solve_many(B, **kw)               # warm-up: buffers and graphs of this width
            ml.solve(B[:, 0], **kw)
            t0 = time.perf_counter()
            singles = [ml.solve(B[:, j], **kw) for j in range(k)]
            t_single = time.perf_counter() - t0
            t0 = time.perf_counter()
            X = ml.solve_many(B, **kw)
            t_many = time.perf_counter() - t0
            col_its = k * its / t_many
            if k == 1:
                base = col_its
            diff = max(float(np.abs(X[:, j] - singles[j]).max()) for j in range(k))
            out[str(k)] = {"column_iterations_per_s": round(col_its, 2), "ratio_vs_k1": round(col_its / base, 3),
                           "speedup_vs_k_single_calls": round(t_single / t_many, 3),
                           "ms_per_batched_iteration": round(1e3 * t_many / its, 3), "max_col_abs_diff_vs_k1": diff}
            bench.log(f"[{name} gmres] k={k}: {out[str(k)]}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="gsnr,jacobi_ne,schwarz")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gmres-maxiter", type=int, default=20)
    ap.add_argument("--grid", type=int, default=DEFAULT_GRID)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_many_ne_schwarz.py: no CUDA device -- this script measures the GPU only")
    gpu, power = BM.gpu_info()
    tstream = torch.cuda.Stream()
    torch.cuda.set_stream(tstream)
    res = {}
    for name in (w for w in args.workloads.split(",") if w):
        ml = build(name, args.grid, stream=tstream.cuda_stream)
        res[name] = {"n": int(ml.levels[0].A.shape[0]), "cycles": measure_cycles(name, ml, args)}
        if name == "gsnr":
            res[name]["gmres"] = measure_gmres(name, ml, args)
        del ml
    print(json.dumps({"metric": "cycles/s and column-cycles/s of solve_many vs k=1 (normal-equation and Schwarz "
                                "smoothers), column-iterations/s of solve_many(accel='gmres')",
                      "gpu": gpu, "power_limit": power, "grid": args.grid, "steps": args.steps,
                      "warmup": args.warmup, "gmres_maxiter": args.gmres_maxiter, "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
