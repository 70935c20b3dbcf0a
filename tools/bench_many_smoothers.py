#!/usr/bin/env python
"""bench_many_smoothers.py -- throughput of MultilevelSolver.solve_many on the default smoothed-aggregation
hierarchies (block Gauss-Seidel) and on polynomial smoothing, against single-vector cycles.

    python tools/bench_many_smoothers.py [--workloads sa_poisson,sa_elasticity,sa_chebyshev] [--steps 10] [--warmup 3]
                                         [--cg-maxiter 20] [--grid N] [--profile DIR]

Workloads, built by this repository's host setup (np.random.seed and right-hand sides from bench.SEED):
    sa_poisson     poisson((2000, 2000)),  smoothed_aggregation_solver(A) carrying the smoother objects of a hierarchy
                   adopted from the reference: symmetric block Gauss-Seidel with blocksize 1 (this repository's own
                   setup installs plain Gauss-Seidel for blocksize 1, which solve_many batched already)
    sa_elasticity  linear_elasticity((300, 300)), smoothed_aggregation_solver(A, B=B): symmetric block Gauss-Seidel,
                   blocksize 2 on the fine level and 3 below
    sa_chebyshev   poisson((2000, 2000)),  smoothed_aggregation_solver(A) with degree-3 Chebyshev pre and post

For each workload and k in {1, 2, 4, 8}:
  * cycles: k columns of B and X resident in HBM, `steps` V-cycles each followed by the per-column residual norm,
    timed with CUDA events after `warmup` cycles (k = 1 amgb_solve_device, k > 1 amgb_solve_many_device);
    column-cycles/s, its ratio to k = 1, and the largest absolute per-column difference between the batched iterate
    and k = 1 runs of the same columns after 2 cycles (it must be 0);
  * CG: k calls of solve(b_j, accel='cg', tol=0, maxiter=ITS) against one solve_many(B, accel='cg', ...) on host
    blocks, host wall clock around each call (both end in a device-to-host copy and a synchronise);
    column-iterations/s, its ratio to k = 1, the speed-up over the k single calls and the largest difference.
Prints one JSON line, with the card's name and power limit (a read-only nvidia-smi query).

--profile DIR: instead, a torch.profiler run of 3 un-timed cycles per workload at k = 1 and k = 4; writes
DIR/bench_many_smoothers_kernels.json with the CUDA time per kernel name.
--grid N: grid edge instead of 2000 / 300 (a quick run; the numbers of DESIGN 5e are at the default sizes).
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

import bench_many as BM  # noqa: E402  (device-block cycling, byte model, card query, kernel table)
from bench_many import bench  # noqa: E402

KS = BM.KS
DEFAULT_GRID = {"sa_poisson": 2000, "sa_elasticity": 300, "sa_chebyshev": 2000}


def build(name, grid, stream=None):
    from pyamg_b200.aggregation import smoothed_aggregation_solver
    from pyamg_b200.gallery import linear_elasticity, poisson
    np.random.seed(bench.SEED)
    t0 = time.time()
    if name == "sa_poisson":
        from functools import partial, update_wrapper
        from pyamg_b200.relaxation import relaxation
        ml = smoothed_aggregation_solver(poisson((grid, grid)), stream=stream)
        sm = partial(relaxation.block_gauss_seidel, iterations=1, sweep="symmetric", blocksize=1)
        update_wrapper(sm, relaxation.block_gauss_seidel)
        for lvl in ml.levels[:-1]:
            lvl.presmoother = lvl.postsmoother = sm
        ml._invalidate()
    elif name == "sa_elasticity":
        A, B = linear_elasticity((grid, grid))
        ml = smoothed_aggregation_solver(A, B=B, stream=stream)
    elif name == "sa_chebyshev":
        sm = ("chebyshev", {"degree": 3, "iterations": 1})
        ml = smoothed_aggregation_solver(poisson((grid, grid)), presmoother=sm, postsmoother=sm, stream=stream)
    else:
        sys.exit(f"bench_many_smoothers.py: unknown workload {name!r}")
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
        nbytes = BM.cycle_bytes(ml, k)
        X2 = torch.zeros((n, k), dtype=torch.float64, device=dev)       # parity: 2 cycles from zero
        BM.run_cycles(E, ml, k, B, X2, 2, norms)
        launches = ml.last_launches()            # 2 cycles with their residual norms, plus the load and store
        diff = 0.0
        for j in range(k):
            xj = torch.zeros(n, dtype=torch.float64, device=dev)
            BM.run_cycles(E, ml, 1, B[:, j].contiguous(), xj, 2, norms)
            torch.cuda.synchronize()
            diff = max(diff, float((X2[:, j] - xj).abs().max()))
        out[str(k)] = {"cycles_per_s": round(cps, 2), "column_cycles_per_s": round(k * cps, 2),
                       "ratio_vs_k1": round(k * cps / base, 3), "ms_per_cycle": round(ms, 3),
                       "launches_per_2_cycles": launches,
                       "alg_GB_per_cycle": round(nbytes / 1e9, 4), "TBps": round(nbytes / (ms * 1e-3) / 1e12, 3),
                       "max_col_abs_diff_vs_k1": diff}
        bench.log(f"[{name}] k={k}: {out[str(k)]}")
    return out


def measure_cg(name, ml, args):
    n = ml.levels[0].A.shape[0]
    its = args.cg_maxiter
    Bfull = np.random.default_rng(bench.SEED).random((n, max(KS)))
    kw = dict(accel="cg", tol=0, maxiter=its)
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
            bench.log(f"[{name} cg] k={k}: {out[str(k)]}")
    return out


def profile(name, ml):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    from pyamg_b200 import _engine as E
    n = ml.levels[0].A.shape[0]
    dev = torch.device("cuda")
    table = {}
    for k in (1, 4):
        B = torch.rand((n, k), dtype=torch.float64, device=dev)
        X = torch.zeros((n, k), dtype=torch.float64, device=dev)
        norms = torch.zeros(16 * k, dtype=torch.float64, device=dev)
        BM.run_cycles(E, ml, k, B, X, 2, norms)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            BM.run_cycles(E, ml, k, B, X, 3, norms)
            torch.cuda.synchronize()
        table[str(k)] = BM._kernel_table(prof, 3, "cycle")
    return table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="sa_poisson,sa_elasticity,sa_chebyshev")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cg-maxiter", type=int, default=20)
    ap.add_argument("--grid", type=int, default=None)
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_many_smoothers.py: no CUDA device -- this script measures the GPU only")
    gpu, power = BM.gpu_info()
    tstream = torch.cuda.Stream()
    torch.cuda.set_stream(tstream)
    res = {}
    for name in (w for w in args.workloads.split(",") if w):
        ml = build(name, args.grid or DEFAULT_GRID[name], stream=tstream.cuda_stream)
        if args.profile:
            res[name] = profile(name, ml)
            continue
        from pyamg_b200 import _engine as E
        res[name] = {"n": int(ml.levels[0].A.shape[0]), "cycles": measure_cycles(name, ml, args),
                     "cg": measure_cg(name, ml, args),
                     "hbm_bytes_after_all_widths": int(E.lib().amgb_hierarchy_device_bytes(ml.handle))}
        del ml
    if args.profile:
        os.makedirs(args.profile, exist_ok=True)
        with open(os.path.join(args.profile, "bench_many_smoothers_kernels.json"), "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps({"gpu": gpu, "power_limit": power, "profile": res}), flush=True)
        return
    print(json.dumps({"metric": "column-cycles/s of solve_many and column-iterations/s of solve_many(accel='cg') "
                                "vs k=1", "gpu": gpu, "power_limit": power, "steps": args.steps,
                      "warmup": args.warmup, "cg_maxiter": args.cg_maxiter, "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
