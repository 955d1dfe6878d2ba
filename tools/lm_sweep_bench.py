#!/usr/bin/env python
"""Sweep of the LM weights against one decode per pair: BASELINE config 5 ([64 x T=1000 x V=29], beam 100, the
reference's test.arpa) with the device scorer, for P (alpha, beta) pairs, two ways:

  sweep           one CTCBeamDecoder.decode_sweep call (ctcdec_decode_batch_lm_sweep_async): one vocabulary scan,
                  P x 64 beam CTAs, one read-out
  sequential      P asynchronous decodes (non_blocking=True, ctcdec_decode_batch_lm_device_async), each after
                  reset_params with its pair

    python tools/lm_sweep_bench.py [--pairs 1,2,4,8,16] [--reps N] [--device I]

For each P both arms are warmed up, then timed N times in alternating rounds with a host clock around the call and a
device synchronise after it.  Prints one JSON line per P: the median and the spread of the call time of each arm,
whether every slice of the sweep equals the sequential decode of its pair bit for bit, and the card and its power
limit, read in the same run.  Writes nothing to disk.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import CONFIGS, L29, TINY_LM, c5_inputs  # noqa: E402
from ctcdecode_b200 import CTCBeamDecoder  # noqa: E402
from tools.lm_device_bench import identical  # noqa: E402
from tools.stream_bench import card_info  # noqa: E402


def pairs_of(P):
    """P distinct pairs around config 5's (2.0, 1.0), alpha = 0 and a negative beta among them"""
    return [(0.25 * (p % 9), 1.0 - 0.5 * (p // 9) - 0.25 * (p % 3)) for p in range(P)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,2,4,8,16", help="comma-separated sweep sizes P")
    ap.add_argument("--reps", type=int, default=5, help="timed calls per arm and P")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    cfg = CONFIGS["c5"]
    B, T = cfg["B"], cfg["T"]
    x = c5_inputs(B, T, 0).to(dev)
    card = card_info(args.device)
    dec = CTCBeamDecoder(L29, model_path=TINY_LM, alpha=cfg["alpha"], beta=cfg["beta"], beam_width=cfg["beam"],
                         cutoff_top_n=cfg["cutoff_top_n"], cutoff_prob=cfg["cutoff_prob"], scorer_provider="device",
                         device_outputs=True, non_blocking=True)
    for P in [int(v) for v in args.pairs.split(",")]:
        pairs = pairs_of(P)
        al, be = [a for a, _ in pairs], [b for _, b in pairs]

        def sweep():
            t0 = time.perf_counter()
            res = dec.decode_sweep(x, al, be)
            torch.cuda.synchronize(dev)
            dt = time.perf_counter() - t0
            return dt, [[r[p].cpu() for r in res] + [dec.last_n_results[p].cpu(), dec.last_flags[p].cpu()]
                        for p in range(P)]

        def sequential():
            t0 = time.perf_counter()
            res = []
            for a, b in pairs:
                dec.reset_params(a, b)
                res.append(list(dec.decode(x)) + [dec.last_n_results, dec.last_flags])
            torch.cuda.synchronize(dev)
            dt = time.perf_counter() - t0
            return dt, [[r.cpu() for r in one] for one in res]

        arms = {"sweep": sweep, "sequential": sequential}
        for fn in arms.values():
            fn()
            fn()  # warm-up: workspace, tables, kernel attributes
        times, outs = {k: [] for k in arms}, {}
        for _ in range(args.reps):
            for k, fn in arms.items():
                dt, outs[k] = fn()
                times[k].append(dt)
        same = all(identical(outs["sweep"][p], outs["sequential"][p]) for p in range(P))
        legs = {k: {"ms_median": 1e3 * statistics.median(t), "ms_min": 1e3 * min(t), "ms_max": 1e3 * max(t),
                    "calls": len(t)} for k, t in times.items()}
        print(json.dumps({"workload": cfg["name"].replace("KenLM scorer hook", "device n-gram scorer"), "P": P,
                          "ctas": P * B, "card": card, "arms": legs,
                          "speedup_median": legs["sequential"]["ms_median"] / legs["sweep"]["ms_median"],
                          "all_slices_identical": bool(same),
                          "note": "host clock around each call and a device synchronise after it; arms alternate "
                                  "within each round"}), flush=True)
        assert same, "P = %d: a slice of the sweep differs from its sequential decode" % P
    dec.reset_params(cfg["alpha"], cfg["beta"])


if __name__ == "__main__":
    main()
