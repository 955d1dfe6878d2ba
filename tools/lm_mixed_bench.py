#!/usr/bin/env python
"""A batch spread over S language models, one mixed call against one call per model: BASELINE config 5's shape
([64 x T=1000 x V=29], beam 100) with the device scorer, utterance b taking model b % S of
  test.arpa (alpha 2.0, beta 1.0), test.arpa (0.5, 2.0), tiny_lm (2.0, 1.0), a KenLM trie of test.arpa (1.0, 0.5)
(the trie needs oracle/_ref/build_binary; without it the fourth model is test.arpa's text again, a distinct scorer).

  mixed           one CTCBeamDecoder.decode_mixed call (ctcdec_decode_batch_lm_mixed_async)
  per_model       S asynchronous decodes (non_blocking=True) of each model's sub-batch on one stream

    python tools/lm_mixed_bench.py [--models 1,2,4] [--per-model 0] [--reps N] [--device I]

--per-model U > 0 gives each model U utterances (B = S x U) instead of spreading 64.  Both arms are warmed up, then
timed N times in alternating rounds with a host clock around the call and a device synchronise after it.  Prints one
JSON line per S: the median and the range of each arm, whether every utterance of the mixed call equals its per-model
decode bit for bit, and the card and its power limit, read in the same run.  Writes only under a temporary directory.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import CONFIGS, L29, c5_inputs  # noqa: E402
from ctcdecode_b200 import CTCBeamDecoder  # noqa: E402
from tools.lm_device_bench import identical  # noqa: E402
from tools.stream_bench import card_info  # noqa: E402

TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
TINY_LM = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
BUILD_BINARY = os.path.join(ROOT, "oracle", "_ref", "build_binary")


def models(tmp):
    trie = TEST_ARPA
    if os.path.exists(BUILD_BINARY):
        trie = os.path.join(tmp, "test.arpa.trie")
        subprocess.run([BUILD_BINARY, "-S", "64M", "-T", tmp, "trie", TEST_ARPA, trie], check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return [(TEST_ARPA, 2.0, 1.0), (TEST_ARPA, 0.5, 2.0), (TINY_LM, 2.0, 1.0), (trie, 1.0, 0.5)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="1,2,4", help="comma-separated model counts S")
    ap.add_argument("--per-model", type=int, default=0, help="utterances per model (0: spread 64 over the models)")
    ap.add_argument("--reps", type=int, default=7, help="timed calls per arm and S")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    cfg = CONFIGS["c5"]
    card = card_info(args.device)
    with tempfile.TemporaryDirectory() as tmp:
        specs = models(tmp)
        decs = [CTCBeamDecoder(L29, model_path=m, alpha=a, beta=b, beam_width=cfg["beam"],
                               cutoff_top_n=cfg["cutoff_top_n"], cutoff_prob=cfg["cutoff_prob"],
                               scorer_provider="device", device_outputs=True, non_blocking=True) for m, a, b in specs]
        for S in [int(v) for v in args.models.split(",")]:
            B = S * args.per_model if args.per_model else cfg["B"]
            T = cfg["T"]
            x = c5_inputs(B, T, 0).to(dev)
            lm_index = torch.arange(B, dtype=torch.int32) % S
            rows = [torch.nonzero(lm_index == s).flatten().to(dev) for s in range(S)]
            subs = [x.index_select(0, r) for r in rows]
            use = decs[:S]

            def mixed():
                t0 = time.perf_counter()
                res = use[0].decode_mixed(x, lm_index, use)
                torch.cuda.synchronize(dev)
                dt = time.perf_counter() - t0
                out = list(res) + [use[0].last_n_results, use[0].last_flags]
                return dt, [[r.index_select(0, rows[s]).cpu() for r in out] for s in range(S)]

            def per_model():
                t0 = time.perf_counter()
                res = []
                for s in range(S):
                    res.append(list(use[s].decode(subs[s])) + [use[s].last_n_results, use[s].last_flags])
                torch.cuda.synchronize(dev)
                dt = time.perf_counter() - t0
                return dt, [[r.cpu() for r in one] for one in res]

            arms = {"mixed": mixed, "per_model": per_model}
            for fn in arms.values():
                fn()
                fn()  # warm-up: workspaces, tables, kernel attributes
            times, outs = {k: [] for k in arms}, {}
            for _ in range(args.reps):
                for k, fn in arms.items():
                    dt, outs[k] = fn()
                    times[k].append(dt)
            same = all(identical(outs["mixed"][s], outs["per_model"][s]) for s in range(S))
            legs = {k: {"ms_median": 1e3 * statistics.median(t), "ms_min": 1e3 * min(t), "ms_max": 1e3 * max(t),
                        "calls": len(t)} for k, t in times.items()}
            print(json.dumps({"workload": "config 5 shape, device n-gram scorer, %d models" % S, "S": S, "B": B,
                              "models": [(os.path.basename(m), a, b) for m, a, b in specs[:S]], "card": card,
                              "arms": legs,
                              "speedup_median": legs["per_model"]["ms_median"] / legs["mixed"]["ms_median"],
                              "all_utterances_identical": bool(same),
                              "note": "host clock around each call and a device synchronise after it; arms alternate "
                                      "within each round"}), flush=True)
            assert same, "S = %d: an utterance of the mixed call differs from its per-model decode" % S


if __name__ == "__main__":
    main()
