#!/usr/bin/env python
"""Streaming arena compaction benchmark (OnlineCTCBeamDecoder.compact): B long streams (beam 100, 29 labels,
ctc-like posteriors) decoded in CUDA chunks of F frames, one arm compacted after every N chunks and one never, the two
arms' chunk calls alternating.  Reports

  bytes        device bytes per stream (DecoderState.device_bytes) after 1k / 10k / 50k frames, per arm
  compact_ms   the time of one compaction call against the frames consumed since the state's last one (the periodic
               calls, and one call on each arm's states at the end of a stream: the never-compacted arm's covers every
               frame)
  chunk_ms     the median chunk-call time per arm (arena growth copies included; the compaction calls are not chunk
               calls and are reported apart)

and, with --lm, the same with the device n-gram scorer of tests/golden/test.arpa.  Times are a host clock around work
that ends in a device synchronise.  The card's name and power limit are read in the same run.  Prints one JSON line;
--out also writes it to a file.

    python tools/stream_compact_bench.py [--frames 50000] [--chunk 250] [--every 4] [--streams 4] [--lm] [--out F]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ctcdecode_b200  # noqa: E402
from ctcdecode_b200.synth import ctc_like_probs  # noqa: E402

L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")


def card_info(index):
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out)
    except (OSError, ValueError, subprocess.TimeoutExpired):
        pass
    return info


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t) * 1e3


def run(args, lm):
    kw = dict(model_path=TEST_ARPA, alpha=1.0, beta=1.0, scorer_provider="device") if lm else {}
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(L29, beam_width=100, device_outputs=True, non_blocking=True, **kw)
    B, T, F = args.streams, args.frames, args.chunk
    probs = ctc_like_probs(B, T, 29, seed=12).cuda()
    arms = {"compacted": [ctcdecode_b200.DecoderState(dec) for _ in range(B)],
            "never": [ctcdecode_b200.DecoderState(dec) for _ in range(B)]}
    chunk_ms = {a: [] for a in arms}
    compact_ms, since = [], 0
    marks = sorted({m for m in (1000, 10000, 50000) if m <= T})
    bytes_at = {a: {} for a in arms}
    dec.decode(probs[:, :F], [ctcdecode_b200.DecoderState(dec) for _ in range(B)], [False] * B)  # warm-up
    for c in range(T // F):
        chunk = probs[:, c * F:(c + 1) * F]
        order = list(arms) if c % 2 == 0 else list(arms)[::-1]
        for a in order:
            _, ms = timed(lambda: dec.decode(chunk, arms[a], [False] * B))
            chunk_ms[a].append(ms)
        since += F
        if (c + 1) % args.every == 0:
            kept, ms = timed(lambda: dec.compact(arms["compacted"]))
            compact_ms.append(dict(frames_since=since, ms=ms, nodes_kept=int(kept.max())))
            since = 0
        done = (c + 1) * F
        for m in marks:
            if done == m:
                for a in arms:
                    bytes_at[a][m] = max(s.device_bytes() for s in arms[a])
    final = {}
    for a in arms:
        fs = since if a == "compacted" else (T // F) * F
        kept, ms = timed(lambda: dec.compact(arms[a]))
        final[a] = dict(frames_since=fs, ms=ms, nodes_kept=int(kept.max()))
    return dict(scorer="test.arpa" if lm else None, streams=B, beam=100, chunk=F, every=args.every,
                bytes_per_stream=bytes_at,
                chunk_ms_median={a: statistics.median(v) for a, v in chunk_ms.items()},
                chunk_ms_max={a: max(v) for a, v in chunk_ms.items()},
                compact_ms_periodic_median=statistics.median([x["ms"] for x in compact_ms]) if compact_ms else None,
                compact_periodic=compact_ms[-3:], compact_final=final)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50000)
    ap.add_argument("--chunk", type=int, default=250)
    ap.add_argument("--every", type=int, default=4)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--lm", action="store_true", help="also run the arm with the device n-gram scorer")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("stream_compact_bench.py needs a GPU")
    torch.cuda.set_device(args.device)
    res = dict(card=card_info(args.device), runs=[run(args, False)] + ([run(args, True)] if args.lm else []))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
