#!/usr/bin/env python
"""Scorer-path benchmark: BASELINE config 5 ([64 x T=1000 x V=29], beam 100, the reference's test.arpa, alpha 2.0,
beta 1.0) through CTCBeamDecoder three ways:

  host            CPU probabilities through the host entry point (ctcdec_decode_batch_lm_host)
  device          CUDA probabilities through the device entry point (ctcdec_decode_batch_lm_device)
  logits_f16      decode_logits of fp16 logits (the device entry, the log-softmax taken by the scan kernel)

    python tools/lm_device_bench.py [--reps N] [--device I] [--scorer hook|device|async] [--model PATH]

--scorer device times the library's own ARPA scorer (scorer_provider="device": the beam kernel computes the LM terms,
no per-frame host handshake) against the hook scorer on the same CUDA probabilities instead:

  hook            the reference's Scorer behind the hook, CUDA probabilities (ctcdec_decode_batch_lm_device)
  ngram           the device scorer, CUDA probabilities (the same entry point)
  ngram_host      the device scorer, CPU probabilities (ctcdec_decode_batch_lm_host)

--scorer async times the device scorer with device outputs three ways, on the same CUDA probabilities:

  blocking        ctcdec_decode_batch_lm_device: the call synchronises and rescores the results on the host
  async           non_blocking=True (ctcdec_decode_batch_lm_device_async): the read-out kernel rescores them
  graph           the async decode captured once into a CUDA graph, replayed

and, in a separate profiled pass afterwards, the CUDA time of the read-out kernel alone (torch.profiler).

--model decodes with another language model than test.arpa, for instance a KenLM binary file written from it by
build_binary (probing or trie): the device scorer and the hook scorer both read it.

Every path is warmed up, then timed N times in alternating rounds with a host clock around the call and a device
synchronise after it.  Prints one JSON line: per path the median and the spread of the call time
and utterances/s; whether the host and device paths gave identical outputs; the card and its power limit, read in the
same run.  Writes nothing to disk.
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
from bench import CONFIGS, L29, PROVIDER, TINY_LM, c5_inputs  # noqa: E402
from ctcdecode_b200 import CTCBeamDecoder  # noqa: E402
from tools.stream_bench import card_info  # noqa: E402


def identical(x, y):
    """bit for bit: n_results, flags, and per row p < n_results the score bits, the length, tokens and timesteps"""
    tok_x, sc_x, ts_x, ln_x, nr_x, fl_x = x
    tok_y, sc_y, ts_y, ln_y, nr_y, fl_y = y
    if not (torch.equal(nr_x, nr_y) and torch.equal(fl_x, fl_y)):
        return False
    for b in range(nr_x.shape[0]):
        n = int(nr_x[b])
        if not (torch.equal(sc_x[b, :n].view(torch.int32), sc_y[b, :n].view(torch.int32)) and
                torch.equal(ln_x[b, :n], ln_y[b, :n])):
            return False
        for p in range(n):
            L = int(ln_x[b, p])
            if not (torch.equal(tok_x[b, p, :L], tok_y[b, p, :L]) and torch.equal(ts_x[b, p, :L], ts_y[b, p, :L])):
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed calls per path")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--scorer", choices=["hook", "device", "async"], default="hook",
                    help="hook: the three input paths of the hook scorer; device: the device scorer against the hook; "
                         "async: the device scorer's blocking, asynchronous and graph-replayed decodes")
    ap.add_argument("--model", default=TINY_LM, help="the language model (ARPA text or a KenLM binary file)")
    args = ap.parse_args()
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    cfg = CONFIGS["c5"]
    B, T = cfg["B"], cfg["T"]
    probs = c5_inputs(B, T, 0)
    probs_d = probs.to(dev)
    logits = probs_d.clamp_min(1e-20).log().mul(1.25).half()
    kw = dict(model_path=args.model, alpha=cfg["alpha"], beta=cfg["beta"], beam_width=cfg["beam"],
              cutoff_top_n=cfg["cutoff_top_n"], cutoff_prob=cfg["cutoff_prob"])
    readout_ms = None
    if args.scorer == "async":
        bdec = CTCBeamDecoder(L29, scorer_provider="device", device_outputs=True, **kw)
        adec = CTCBeamDecoder(L29, scorer_provider="device", device_outputs=True, non_blocking=True, **kw)
        gdec = CTCBeamDecoder(L29, scorer_provider="device", device_outputs=True, non_blocking=True, **kw)
        static = probs_d.clone()
        gdec.decode(static)  # outside the capture first: tables, kernel limits
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            g_out = list(gdec.decode(static)) + [gdec.last_n_results, gdec.last_flags]

        def replay():
            graph.replay()
            return g_out[:4]
        paths = {"blocking": (bdec, lambda: bdec.decode(probs_d)), "async": (adec, lambda: adec.decode(probs_d)),
                 "graph": (gdec, replay)}
        compared = ("blocking", "async")
    else:
        dec = CTCBeamDecoder(L29, scorer_provider=PROVIDER, **kw)
        paths = {"host": (dec, lambda: dec.decode(probs)), "device": (dec, lambda: dec.decode(probs_d)),
                 "logits_f16": (dec, lambda: dec.decode_logits(logits))}
        compared = ("host", "device")
    if args.scorer == "device":
        ndec = CTCBeamDecoder(L29, scorer_provider="device", **kw)
        paths = {"hook": (dec, lambda: dec.decode(probs_d)), "ngram": (ndec, lambda: ndec.decode(probs_d)),
                 "ngram_host": (ndec, lambda: ndec.decode(probs))}
        compared = ("hook", "ngram")

    def call(name):
        d, fn = paths[name]
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize(dev)
        dt = time.perf_counter() - t0
        if name == "graph":
            return dt, [x.cpu() for x in g_out]
        return dt, [x.cpu() for x in res] + [d.last_n_results.cpu(), d.last_flags.cpu()]

    outs, times = {}, {name: [] for name in paths}
    for name in paths:
        for _ in range(2):
            call(name)  # warm-up: workspace, pinned blocks, dictionary upload, kernel attributes, hook caches
    for _ in range(args.reps):
        for name in paths:
            dt, outs[name] = call(name)
            times[name].append(dt)
    legs = {name: {"ms_median": 1e3 * statistics.median(t), "ms_min": 1e3 * min(t), "ms_max": 1e3 * max(t),
                   "utterances_per_s": B / statistics.median(t), "calls": len(t)} for name, t in times.items()}
    same = identical(outs[compared[0]], outs[compared[1]])
    if args.scorer == "device":
        same = same and identical(outs["ngram"], outs["ngram_host"])
    if args.scorer == "async":
        same = same and identical(outs["async"], outs["graph"])
        # the read-out kernel alone, from a profiled pass of its own (the timed rounds above run without the profiler)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                adec.decode(probs_d)
            torch.cuda.synchronize(dev)
        ks = [e.device_time for e in prof.events() if "lm_readout_kernel" in e.name]
        readout_ms = {"ms_median": statistics.median(ks) / 1e3, "ms_min": min(ks) / 1e3, "ms_max": max(ks) / 1e3,
                      "launches": len(ks)} if ks else None
    print(json.dumps({"workload": cfg["name"], "scorer": args.scorer, "model": os.path.basename(args.model),
                      "library": os.environ.get("CTCDECODE_B200_LIB") or "in-tree", "card": card_info(args.device), "paths": legs,
                      "readout_kernel": readout_ms,
                      ("all_arms_identical" if args.scorer == "async" else "%s_%s_identical" % compared): bool(same),
                      "note": "host clock around each call and a device synchronise after it; paths alternate within "
                              "each round"}), flush=True)
    assert same, "%s and %s gave different results" % compared


if __name__ == "__main__":
    main()
