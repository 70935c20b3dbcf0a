"""A/B of two builds of the engine library on one bench.py workload, in one process.

For a change that has no runtime switch (a kernel rewritten in place), build the parent commit's
libpyamg_b200.so somewhere else and pass both.  The hierarchy is set up once; each round uploads it with every
library in turn (each library keeps its own device copy and settings) and times `--steps` device-resident cycles
with the stop-test norms, as bench.py does.  Reports cycles/s per library with min / max over the rounds, the
per-level, per-op profile of one un-graphed cycle of each (ms, charged GB, GB/s), whether the final iterates and
residual norms are bit-identical to the first library's, and the card's name, power limit and max SM clock.

    python tools/ab_builds.py parent=/path/to/parent/libpyamg_b200.so new=tree [--workload cfg3] [--steps 20]
                              [--rounds 3] [--out DIR/ab.json]

`tree` stands for the library of this tree (built if stale).
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+", help="name=path of a libpyamg_b200.so, or name=tree")
    ap.add_argument("--workload", default="cfg3", choices=["cfg3", "cfg2", "cfg4", "cfg5"])
    ap.add_argument("--grid", type=int, default=None, help="default: bench.py's size for the workload")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import bench
    from pyamg_b200 import _engine as E
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    libs = {}
    for spec in args.libs:
        name, path = spec.split("=", 1)
        libs[name] = E.lib() if path == "tree" else E._bind(ctypes.CDLL(os.path.abspath(path)))
    names = list(libs)
    stream = torch.cuda.Stream()                  # the solver's stream (as bench.py): the events below bracket its work
    torch.cuda.set_stream(stream)
    bench.WORKLOAD["name"] = args.workload
    grid = args.grid if args.grid is not None else bench.DEFAULT_GRID[args.workload]
    ml = bench.build_hierarchy((grid,) * 3, stream=stream.cuda_stream)
    n = ml.levels[0].A.shape[0]
    dev = torch.device("cuda", 0)
    b = torch.from_numpy(np.random.default_rng(bench.SEED).random(n)).to(dev)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    owner = None                                  # the library that holds ml's device copy
    rates = {v: [] for v in names}
    prof, outs = {}, {}
    for rnd in range(args.rounds):
        for v in names:
            if owner is not None:
                E._lib = libs[owner]
                ml._invalidate()
            E._lib = libs[v]
            owner = v
            ml.upload()
            L, h = libs[v], ml.handle
            x = torch.zeros(n, dtype=torch.float64, device=dev)
            norms = torch.zeros(args.steps + 2, dtype=torch.float64, device=dev)
            E.check(L.amgb_solve_device(h, P(b), P(x), 3, 0, 1, P(norms)))      # warm-up, graph capture
            x.zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            E.check(L.amgb_solve_device(h, P(b), P(x), args.steps, 0, 1, P(norms)))
            e1.record()
            torch.cuda.synchronize()
            rates[v].append(args.steps / (e0.elapsed_time(e1) * 1e-3))
            print(f"round {rnd} {v}: {rates[v][-1]:.2f} cycles/s", flush=True)
            if rnd == 0:
                outs[v] = (x.cpu().numpy(), np.sqrt(norms[:args.steps + 1].cpu().numpy()))
                ml.profile_cycle()
                recs = np.concatenate([ml.profile_cycle() for _ in range(3)])
                table = {}
                for lvl, op, rows, nnz, nbytes, t in recs:
                    g = table.setdefault(f"L{int(lvl)}:op{int(op)}", [0, 0.0, 0.0])
                    g[0] += 1; g[1] += t; g[2] += nbytes
                prof[v] = {k: {"launches_per_cycle": g[0] // 3, "ms_per_cycle": round(g[1] / 3, 4),
                               "GB_per_cycle": round(g[2] / 3e9, 3), "GBps": round(g[2] / g[1] / 1e6, 1)}
                           for k, g in sorted(table.items())}
                prof[v]["cycle_ms_profiled"] = round(float(recs[:, 5].sum()) / 3, 3)
    E._lib = libs[owner]
    ml._invalidate()
    base = outs[names[0]]
    cmp = {v: {"x_bit_identical": bool(np.array_equal(outs[v][0].view(np.int64), base[0].view(np.int64))),
               "norms_bit_identical": bool(np.array_equal(outs[v][1].view(np.int64), base[1].view(np.int64)))}
           for v in names[1:]}
    summ = {v: {"median": float(np.median(r)), "min": float(np.min(r)), "max": float(np.max(r)), "runs": r}
            for v, r in rates.items()}
    res = {"card": card, "workload": args.workload, "grid": grid, "steps": args.steps, "rates": summ, "profile": prof,
           "compare_to_" + names[0]: cmp}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
