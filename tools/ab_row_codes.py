"""A/B of the row codes on the bench.py headline (256^3 Poisson, RS, symmetric multi-colour GS).

Builds the hierarchy once and alternates uploads with per-entry pair codes (AMGB_NO_ROW_CODES=1) and with row codes,
timing `--steps` device-resident V-cycles with the stop-test norms (what bench.py times) per round.  Reports
V-cycles/s per variant with the spread, the per-level, per-op profile of one cycle of each (a launch is charged the
bytes it streams: 1 B per row plus its tile descriptors and tables when row-coded, 1 B per entry plus 4 B per row
pointer and 16 B per pair when pair-coded), the GB per cycle, the device footprint, whether the final iterates and
residual norms are bit-identical, and the card's name, power limit and max SM clock.  --no-hints runs both variants
without the L2 eviction hints (AMGB_NO_HINTS=1).

    python tools/ab_row_codes.py [--grid 256] [--steps 20] [--rounds 3] [--no-hints] [--out DIR/ab.json]
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
    ap.add_argument("--no-hints", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.no_hints:
        os.environ["AMGB_NO_HINTS"] = "1"
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
    variants = ["pair8", "row8"]
    rates = {v: [] for v in variants}
    prof, outs, footprint = {}, {}, {}
    for rnd in range(args.rounds):
        for v in variants:
            os.environ.pop("AMGB_NO_ROW_CODES", None)
            if v == "pair8":
                os.environ["AMGB_NO_ROW_CODES"] = "1"
            ml._invalidate()
            footprint[v] = ml.upload()
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
                table = {}
                for lvl, op, rows, nnz, nbytes, t in recs:
                    g = table.setdefault(f"L{int(lvl)}:op{int(op)}", [0, 0.0, 0.0])
                    g[0] += 1; g[1] += t; g[2] += nbytes
                prof[v] = {k: {"launches_per_cycle": g[0] // 3, "ms_per_cycle": round(g[1] / 3, 4),
                               "GB_per_cycle": round(g[2] / 3e9, 3), "GBps": round(g[2] / g[1] / 1e6, 1)}
                           for k, g in sorted(table.items())}
                prof[v]["cycle_ms_profiled"] = round(float(recs[:, 5].sum()) / 3, 3)
                prof[v]["algorithmic_GB_per_cycle"] = round(float(recs[:, 4].sum()) / 3e9, 3)
    ml._invalidate()
    base = outs[variants[0]]
    cmp = {}
    for v in variants[1:]:
        cmp[v] = {"x_bit_identical": bool(np.array_equal(outs[v][0].view(np.int64), base[0].view(np.int64))),
                  "norms_bit_identical": bool(np.array_equal(outs[v][1].view(np.int64), base[1].view(np.int64)))}
    summ = {v: {"median": float(np.median(r)), "min": float(np.min(r)), "max": float(np.max(r)), "runs": r}
            for v, r in rates.items()}
    res = {"card": card, "grid": args.grid, "steps": args.steps, "hints": not args.no_hints, "rates": summ,
           "device_bytes": footprint,
           "profile": prof, "compare_to_" + variants[0]: cmp}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
