"""A/B of the last-wave residual on the bench.py headline (256^3 Poisson, RS, symmetric multi-colour GS).

Builds the hierarchy once and alternates uploads with and without it (AMGB_NO_WAVE_RESID=1), timing
`--steps` device-resident V-cycles with the stop-test norms (what bench.py times) per round.  Reports V-cycles/s per
variant with the spread, the level-0 per-launch profile of each, whether the final iterates are bit-identical and
how far the residual norms differ, and the card's name and power limit.

    python tools/ab_wave_residual.py [--grid 256] [--steps 20] [--rounds 3] [--out DIR/ab.json]
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
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import bench
    from pyamg_b200 import _engine as E
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    stream = torch.cuda.Stream()                  # the solver's stream (as bench.py): the events below bracket its work
    torch.cuda.set_stream(stream)
    ml = bench.build_hierarchy((args.grid,) * 3, stream=stream.cuda_stream)
    n = ml.levels[0].A.shape[0]
    dev = torch.device("cuda", 0)
    b = torch.from_numpy(np.random.default_rng(bench.SEED).random(n)).to(dev)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    variants = ["plain", "wave_resid"]
    rates = {v: [] for v in variants}
    prof, outs = {}, {}
    for rnd in range(args.rounds):
        for v in variants:
            os.environ.pop("AMGB_NO_WAVE_RESID", None)
            if v == "plain":
                os.environ["AMGB_NO_WAVE_RESID"] = "1"
            ml._invalidate()
            ml.upload()
            L, h = E.lib(), ml.handle
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
            print(f"round {rnd} {v}: {rates[v][-1]:.2f} V-cycles/s", flush=True)
            if rnd == 0:
                outs[v] = (x.cpu().numpy(), np.sqrt(norms[:args.steps + 1].cpu().numpy()))
                ml.profile_cycle()
                recs = np.concatenate([ml.profile_cycle() for _ in range(3)])
                lv0 = {}
                for lvl, op, rows, nnz, nbytes, t in recs:
                    if int(lvl) != 0:
                        continue
                    g = lv0.setdefault(str(int(op)), [0, 0.0, 0.0])
                    g[0] += 1; g[1] += t; g[2] += nbytes
                prof[v] = {op: {"launches_per_cycle": g[0] // 3, "ms_per_cycle": round(g[1] / 3, 4),
                                "GB_per_cycle": round(g[2] / 3e9, 3), "GBps": round(g[2] / g[1] / 1e6, 1)}
                           for op, g in lv0.items()}
                prof[v]["cycle_ms_profiled"] = round(float(recs[:, 5].sum()) / 3, 3)
    ml._invalidate()
    base = outs[variants[0]]
    cmp = {}
    for v in variants[1:]:
        cmp[v] = {"x_bit_identical": bool(np.array_equal(outs[v][0].view(np.int64), base[0].view(np.int64))),
                  "max_rel_norm_diff": float(np.max(np.abs(outs[v][1] - base[1]) / base[1]))}
    summ = {v: {"mean": float(np.mean(r)), "min": float(np.min(r)), "max": float(np.max(r)), "runs": r}
            for v, r in rates.items()}
    res = {"card": card, "grid": args.grid, "steps": args.steps, "rates": summ, "level0_profile": prof,
           "compare_to_" + variants[0]: cmp}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
