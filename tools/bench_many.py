#!/usr/bin/env python
"""bench_many.py -- throughput of MultilevelSolver.solve_many (amgb_solve_many_device) against single-vector cycles.

    python tools/bench_many.py [--workloads cfg3,cfg2,cfg5] [--steps 10] [--warmup 3] [--profile DIR]
                               [--accel cg|bicgstab|gmres|fgmres|cgnr|cgne|minimal_residual|steepest_descent]
                               [--accel-maxiter 20] [--fallback-its 3] [--cfg9-grid 1000]

For each workload (hierarchies from bench.build_hierarchy at the bench's default sizes) and k in {1, 2, 4, 8}: k
columns of B and X resident in HBM, `steps` V-cycles each followed by the per-column residual norm (what one
iteration of solve does), timed with CUDA events after `warmup` cycles.  k = 1 runs amgb_solve_device, k > 1
amgb_solve_many_device.  Prints one JSON line with, per workload and k: batched cycles/s, column-cycles/s, its ratio
to k = 1 in the same run, the algorithmic bytes of one batched cycle (SURVEY 8(d): 12 B per stored entry + 4 B per
row pointer of every launch of the cycle, plus its vector terms times k) and the achieved TB/s, and the largest
per-column relative difference between the batched iterate and k = 1 runs of the same columns after 2 cycles.

--profile DIR: instead, a torch.profiler run of a few cycles of cfg3 at k = 1 and k = 4 (with --accel: k = 1, 4, 8;
separate from the timed run); writes DIR/bench_many_kernels.json with the CUDA time per kernel name (the batched kernels carry K).

--accel cg|bicgstab|gmres|fgmres: the batched Krylov solve instead of plain cycles.  For each workload and k, k calls of
solve(b_j, accel=..., tol=0, maxiter=ITS) against one solve_many(B, accel=..., tol=0, maxiter=ITS) on host blocks,
timed with the host wall clock around the call (both entries end in a device-to-host copy and a synchronise and move
the same host bytes).  Reports column-iterations/s, its ratio to k = 1, the speed-up over the k single calls, the
algorithmic bytes of one batched iteration (the preconditioning cycles' launch list plus the Krylov SpMVs with the
operator once and the vector terms times k) and the largest per-column relative difference from the single solves;
then one tol = 1e-8 run at k = 8 with both sides' per-column iteration counts (GMRES: at most ITS inner iterations,
which also bounds its reflector store).  The hierarchy's device bytes after the run show which width GMRES ran at
(its reflector store is K x (ITS + 1) x n doubles, twice that for FGMRES).  With --profile: the kernel breakdown of
solve_many(accel=...) at k = 1, 4 and 8 on cfg3.
--accel cgnr|cgne|minimal_residual|steepest_descent also times, at k = 1, the resident solve against the path it
replaced: the reference's host pyamg.krylov.<accel> (from oracle/_ref/site) with the GPU cycle as M, FALLBACK_ITS
iterations each.  Workload cfg9 is the reference's AIR hierarchy of 2-D upwind advection on a CFG9_GRID^2 grid.
Needs an NVIDIA GPU: without one the script exits with an error, there is no CPU timing.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definitions and sizes)

KS = (1, 2, 4, 8)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power = (out[0].split(",") + ["?"])[:2] if out else ("?", "?")
    return name.strip(), power.strip()


def cycle_bytes(ml, k):
    """Algorithmic bytes of one cycle on k columns: operator part once, vector part k times."""
    recs = ml.profile_cycle()
    total = 0.0
    for _lvl, _op, rows, nnz, nbytes, _ms in recs:
        op_bytes = 12.0 * nnz + 4.0 * (rows + 1)
        total += op_bytes + k * max(nbytes - op_bytes, 0.0)
    return total


def run_cycles(E, ml, k, B, X, ncyc, norms):
    P = lambda t: ctypes.c_void_p(t.data_ptr())      # noqa: E731
    if k == 1:
        E.check(E.lib().amgb_solve_device(ml.handle, P(B), P(X), ncyc, 0, 1, P(norms)))
    else:
        E.check(E.lib().amgb_solve_many_device(ml.handle, k, P(B), P(X), ncyc, 0, 1, P(norms)))


def measure(name, args, tstream):
    import torch
    from pyamg_b200 import _engine as E
    bench.WORKLOAD["name"] = name
    g = bench.DEFAULT_GRID[name]
    ml = bench.build_hierarchy((g,) * 3, stream=tstream.cuda_stream)
    ml.upload()
    n = ml.levels[0].A.shape[0]
    dev = torch.device("cuda")
    rng = np.random.default_rng(bench.SEED)
    Bfull = torch.from_numpy(rng.random((n, max(KS)))).to(dev)
    out = {}
    base = None
    for k in KS:
        B = Bfull[:, :k].contiguous()
        X = torch.zeros((n, k), dtype=torch.float64, device=dev)
        norms = torch.zeros((args.steps + args.warmup + 1) * k, dtype=torch.float64, device=dev)
        run_cycles(E, ml, k, B, X, args.warmup, norms)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run_cycles(E, ml, k, B, X, args.steps, norms)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        cps = 1e3 / ms
        if k == 1:
            base = cps
        nbytes = cycle_bytes(ml, k)
        # parity: 2 cycles from zero, batched versus one column at a time
        X2 = torch.zeros((n, k), dtype=torch.float64, device=dev)
        run_cycles(E, ml, k, B, X2, 2, norms)
        diff = 0.0
        for j in range(k):
            bj = B[:, j].contiguous()
            xj = torch.zeros(n, dtype=torch.float64, device=dev)
            run_cycles(E, ml, 1, bj, xj, 2, norms)
            torch.cuda.synchronize()
            diff = max(diff, float(torch.linalg.norm(X2[:, j] - xj) / torch.linalg.norm(xj)))
        out[str(k)] = {"cycles_per_s": round(cps, 2), "column_cycles_per_s": round(k * cps, 2),
                       "ratio_vs_k1": round(k * cps / base, 3), "ms_per_cycle": round(ms, 3),
                       "alg_GB_per_cycle": round(nbytes / 1e9, 4), "TBps": round(nbytes / (ms * 1e-3) / 1e12, 3),
                       "max_col_rel_diff_vs_k1": diff}
        bench.log(f"[{name}] k={k}: {out[str(k)]}")
        del B, X, X2, norms
    out["n"] = int(n)
    out["hbm_bytes_after_all_widths"] = int(E.lib().amgb_hierarchy_device_bytes(ml.handle))
    return out


# vector passes of one Krylov iteration besides the preconditioning cycles, in bytes per row and column: SpMV x in and
# y out (16 B), a dot product (16 B), an axpby (24 B), a block copy (16 B), the zero fill of the cycle's iterate (8 B)
# (a residual b - A x: 24 B).  CGNR / CGNE: one cycle, A and A^H once each (A^H has the nnz of A), three dot products,
# three axpbys; minimal residual: two cycles (it recomputes r and M r on all but every 50th step), A z and a residual,
# three dot products, one axpby and a copy of M r; steepest descent: one cycle, A z and a residual, three dot products
# and one axpby (pyamg/krylov/_cgnr.py, _cgne.py, _minimal_residual.py, _steepest_descent.py; abi_krylov_more.cuh)
KRYLOV_PASSES = {"cg": dict(cycles=1, spmv=1, vec=16 + 3 * 16 + 3 * 24 + 8),
                 "bicgstab": dict(cycles=2, spmv=2, vec=2 * 16 + 5 * 16 + 6 * 24 + 4 * 16 + 2 * 8),
                 "cgnr": dict(cycles=1, spmv=2, vec=2 * 16 + 3 * 16 + 3 * 24 + 8),
                 "cgne": dict(cycles=1, spmv=2, vec=2 * 16 + 3 * 16 + 3 * 24 + 8),
                 "minimal_residual": dict(cycles=2, spmv=2, vec=16 + 24 + 3 * 16 + 24 + 16 + 2 * 8),
                 "steepest_descent": dict(cycles=1, spmv=2, vec=16 + 24 + 3 * 16 + 24 + 8)}
MORE = ("cgnr", "cgne", "minimal_residual", "steepest_descent")


def build(name, cfg9_grid):
    """bench's hierarchy of `name` at its default size; cfg9: the reference's AIR hierarchy of 2-D upwind advection
    (tests/golden/make_golden.py's cfg9 at cfg9_grid^2 unknowns), set up by the reference from oracle/_ref/site."""
    if name != "cfg9":
        bench.WORKLOAD["name"] = name
        g = bench.DEFAULT_GRID[name]
        return bench.build_hierarchy((g,) * 3)
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref", "site"))
    import pyamg
    from pyamg.gallery import advection_2d
    from pyamg_b200 import MultilevelSolver
    A, _ = advection_2d((cfg9_grid, cfg9_grid), theta=np.pi / 5.0)
    return MultilevelSolver.from_pyamg(pyamg.air_solver(A.tocsr()))


CFG9_GRID = 1000


def fallback_versus_resident(ml, accel, its):
    """One solve(b, accel=..., tol=0, maxiter=its) resident against the path it replaces: the reference's host
    pyamg.krylov.<accel> with the GPU cycle as M (two n-vector copies per cycle), both timed on the host clock."""
    import time
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref", "site"))
    from pyamg import krylov as ref_krylov
    A = ml.levels[0].A
    b = np.random.default_rng(bench.SEED).random(A.shape[0])
    ml.solve(b, accel=accel, tol=0, maxiter=1)
    t0 = time.perf_counter()
    x = ml.solve(b, accel=accel, tol=0, maxiter=its)
    t_res = time.perf_counter() - t0
    M = ml.aspreconditioner()
    t0 = time.perf_counter()
    xr, _ = getattr(ref_krylov, accel)(A, b, tol=0, maxiter=its, M=M)
    t_ref = time.perf_counter() - t0
    return {"iterations": its, "ms_per_iteration_resident": round(1e3 * t_res / its, 2),
            "ms_per_iteration_host_fallback": round(1e3 * t_ref / its, 2), "speedup": round(t_ref / t_res, 2),
            "rel_diff": float(np.linalg.norm(x - xr) / max(np.linalg.norm(xr), 1e-300))}



def gmres_vector_bytes(its, flexible):
    """Vector bytes per row and column of one GMRES inner iteration, averaged over `its` of them: inner iteration j
    makes 2j + 2 reflections (a dot product, 16 B, and an axpy, 24 B), plus the unit reflector (16 B), the next
    reflector with its norm and divide (3 x 16 B), the tail norm (8 B), the gathers into and out of the level
    numbering (2 x 16 B) and the cycle's zero fill (8 B); FGMRES also stores the preconditioned direction (16 B)."""
    return (its + 1) * 40 + 16 + 48 + 8 + 32 + 8 + (16 if flexible else 0)


def krylov_iteration_bytes(ml, accel, k, its):
    """Algorithmic bytes of one batched Krylov iteration on k columns: operator part once, vector part k times."""
    if accel in ("gmres", "fgmres"):
        m = dict(cycles=1, spmv=1, vec=gmres_vector_bytes(its, accel == "fgmres"))
    else:
        m = KRYLOV_PASSES[accel]
    A = ml.levels[0].A
    n = A.shape[0]
    spmv_op = 12.0 * A.nnz + 4.0 * (n + 1)
    return m["cycles"] * cycle_bytes(ml, k) + m["spmv"] * spmv_op + k * m["vec"] * float(n)


def measure_accel(name, args):
    import time
    import warnings
    from pyamg_b200 import _engine as E
    ml = build(name, args.cfg9_grid)
    ml.upload()
    n = ml.levels[0].A.shape[0]
    its = args.accel_maxiter
    Bfull = np.random.default_rng(bench.SEED).random((n, max(KS)))
    kw = dict(accel=args.accel, tol=0, maxiter=its)
    out = {}
    base = None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # non-symmetric smoother pairs warn under CG, as in solve
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
            nbytes = krylov_iteration_bytes(ml, args.accel, k, its)
            diff = max(float(np.linalg.norm(X[:, j] - singles[j]) / np.linalg.norm(singles[j])) for j in range(k))
            out[str(k)] = {"column_iterations_per_s": round(col_its, 2), "ratio_vs_k1": round(col_its / base, 3),
                           "speedup_vs_k_single_calls": round(t_single / t_many, 3),
                           "ms_per_batched_iteration": round(1e3 * t_many / its, 3),
                           "alg_GB_per_batched_iteration": round(nbytes / 1e9, 4),
                           "TBps": round(nbytes * its / t_many / 1e12, 3), "max_col_rel_diff_vs_k1": diff}
            bench.log(f"[{name} {args.accel}] k={k}: {out[str(k)]}")
        # a tolerance run at k = 8: every column's iteration count equals its single solve's
        B = np.ascontiguousarray(Bfull[:, :8])
        tkw = dict(accel=args.accel, tol=1e-8,
                   maxiter=its if args.accel in ("gmres", "fgmres") else (2 * its if args.accel in MORE else 200))
        res = []
        X, info = ml.solve_many(B, residuals=res, return_info=True, **tkw)
        its_single, diff = [], 0.0
        for j in range(8):
            rj = []
            xj = ml.solve(B[:, j], residuals=rj, **tkw)
            its_single.append(len(rj) - 1)
            diff = max(diff, float(np.linalg.norm(X[:, j] - xj) / np.linalg.norm(xj)))
        out["tol1e-8_k8"] = {"iterations_batched": [len(r) - 1 for r in res], "iterations_single": its_single,
                             "info": [int(i) for i in info], "max_col_rel_diff_vs_k1": diff}
        if args.accel in MORE and args.fallback_its > 0:
            out["fallback_k1"] = fallback_versus_resident(ml, args.accel, args.fallback_its)
            bench.log(f"[{name} {args.accel}] fallback: {out['fallback_k1']}")
    out["n"] = int(n)
    out["hbm_bytes_after_all_widths"] = int(E.lib().amgb_hierarchy_device_bytes(ml.handle))
    return out


def _kernel_table(prof, per, unit):
    rows = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t > 0:
            rows[ev.key] = {"us_per_" + unit: round(t / per, 1), "calls_per_" + unit: ev.count / per}
    return dict(sorted(rows.items(), key=lambda kv: -kv[1]["us_per_" + unit])[:25])


def profile(args, tstream):
    import torch
    import warnings
    from torch.profiler import ProfilerActivity, profile as tprofile
    from pyamg_b200 import _engine as E
    bench.WORKLOAD["name"] = "cfg3"
    g = bench.DEFAULT_GRID["cfg3"]
    ml = bench.build_hierarchy((g,) * 3, stream=None if args.accel else tstream.cuda_stream)
    ml.upload()
    n = ml.levels[0].A.shape[0]
    dev = torch.device("cuda")
    table = {}
    for k in ((1, 4, 8) if args.accel else (1, 4)):
        if args.accel:                   # per Krylov iteration of solve_many(accel=...)
            B = np.random.default_rng(k).random((n, k))
            kw = dict(accel=args.accel, tol=0, maxiter=5)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                ml.solve_many(B, **kw)
                with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                    ml.solve_many(B, **kw)
            table[str(k)] = _kernel_table(prof, 5, "iteration")
            table[str(k)]["hbm_bytes"] = int(E.lib().amgb_hierarchy_device_bytes(ml.handle))
            continue
        B = torch.rand((n, k), dtype=torch.float64, device=dev)
        X = torch.zeros((n, k), dtype=torch.float64, device=dev)
        norms = torch.zeros(16 * k, dtype=torch.float64, device=dev)
        run_cycles(E, ml, k, B, X, 2, norms)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            run_cycles(E, ml, k, B, X, 3, norms)
            torch.cuda.synchronize()
        table[str(k)] = _kernel_table(prof, 3, "cycle")
    os.makedirs(args.profile, exist_ok=True)
    with open(os.path.join(args.profile, "bench_many_kernels.json"), "w") as f:
        json.dump(table, f, indent=1)
    return table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2,cfg5")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", default=None, metavar="DIR")
    ap.add_argument("--accel", default=None, choices=("cg", "bicgstab", "gmres", "fgmres") + MORE)
    ap.add_argument("--fallback-its", type=int, default=3)
    ap.add_argument("--cfg9-grid", type=int, default=CFG9_GRID)
    ap.add_argument("--accel-maxiter", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_many.py: no CUDA device -- this script measures the GPU only")
    name, power = gpu_info()
    tstream = torch.cuda.Stream()
    torch.cuda.set_stream(tstream)
    if args.profile:
        table = profile(args, tstream)
        print(json.dumps({"gpu": name, "power_limit": power, "accel": args.accel, "profile": table}), flush=True)
        return
    if args.accel:
        res = {w: measure_accel(w, args) for w in args.workloads.split(",") if w}
        print(json.dumps({"metric": f"column-iterations/s of solve_many(accel='{args.accel}') vs k=1", "gpu": name,
                          "power_limit": power, "maxiter": args.accel_maxiter, "workloads": res}), flush=True)
        return
    res = {w: measure(w, args, tstream) for w in args.workloads.split(",") if w}
    print(json.dumps({"metric": "column-cycles/s of solve_many vs k=1", "gpu": name, "power_limit": power,
                      "steps": args.steps, "warmup": args.warmup, "workloads": res}), flush=True)


if __name__ == "__main__":
    main()
