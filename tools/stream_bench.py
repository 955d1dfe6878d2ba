#!/usr/bin/env python
"""Streaming benchmark: the config-2 batch ([256 x T=1000 x V=29], beam 100, cutoff_top_n 40) decoded by
OnlineCTCBeamDecoder in chunks of N frames, three ways:

  host              CPU chunks through the host entry point (ctcdec_decode_stream_host)
  device            CUDA chunks through the device entry point (ctcdec_decode_stream_device), results left on the GPU
  device+committed  the same, plus a committed-prefix read-out (OnlineCTCBeamDecoder.committed_prefix) after every chunk

    python tools/stream_bench.py [--chunk N] [--device I]

Prints one JSON line: per path the time per chunk call (wall clock; the device paths synchronise after every chunk,
the host path returns synchronised) and utterances/s over the whole stream; whether the three final outputs are
identical; and the committed-prefix kernel's time beside an eos read-out (mostly the finalize kernel) of the same
states after 100, 500 and 1000 frames (CUDA events).  The card and its power limit are reported with the numbers.
Writes nothing to disk.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctcdecode_b200  # noqa: E402
from ctcdecode_b200 import _native  # noqa: E402
from ctcdecode_b200.synth import ctc_like_probs  # noqa: E402

CFG = dict(B=256, T=1000, V=29, beam=100, cutoff_top_n=40, cutoff_prob=1.0)


def card_info(index):
    """Name and power limit of the GPU (read-only nvidia-smi query; None where unavailable)."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def stream_leg(lib, dev, local_rank, chunk):
    """The config-2 batch through OnlineCTCBeamDecoder in chunks of `chunk` frames, three ways (see the module doc)."""
    B, T, V, Kb = CFG["B"], CFG["T"], CFG["V"], CFG["beam"]
    probs = ctc_like_probs(B, T, V, seed=0)
    probs_d = probs.to(dev)
    cuts = list(range(0, T, chunk)) + [T]
    labels = [str(i) for i in range(V)]

    def run(path):
        dec = ctcdecode_b200.OnlineCTCBeamDecoder(labels, beam_width=Kb, cutoff_top_n=CFG["cutoff_top_n"],
                                                  cutoff_prob=CFG["cutoff_prob"], device=dev,
                                                  device_outputs=path != "host")
        states = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
        times, res, since = [], None, None
        torch.cuda.synchronize(dev)
        t_all = time.perf_counter()
        for a, b in zip(cuts[:-1], cuts[1:]):
            eos = [b == T] * B
            t0 = time.perf_counter()
            if path == "host":
                res = dec.decode(probs[:, a:b], states, eos)
            else:
                res = dec.decode(probs_d[:, a:b], states, eos)
                if path == "device+committed":
                    since = dec.committed_prefix(states, since)[3]  # (waits for the device: sizes the new part)
                torch.cuda.synchronize(dev)
            times.append(time.perf_counter() - t0)
        total = time.perf_counter() - t_all
        out = [x.cpu() for x in res] + [dec.last_n_results.cpu(), dec.last_flags.cpu()]
        for s in states:
            s.release()
        return times, total, out

    legs, outs = {}, {}
    for path in ("host", "device", "device+committed"):
        run(path)  # warm-up (workspace, kernel attributes, pinned buffers)
        times, total, outs[path] = run(path)
        legs[path] = {"chunk_calls": len(times), "ms_per_chunk_mean": 1e3 * statistics.mean(times),
                      "ms_per_chunk_median": 1e3 * statistics.median(times), "ms_whole_stream": 1e3 * total,
                      "utterances_per_s": B / total}

    def same(x, y):
        tok_x, sc_x, ts_x, ln_x, nr_x, fl_x = x
        tok_y, sc_y, ts_y, ln_y, nr_y, fl_y = y
        if not (torch.equal(nr_x, nr_y) and torch.equal(fl_x, fl_y) and torch.equal(ln_x, ln_y)):
            return False
        for b in range(B):
            n = int(nr_x[b])
            if not torch.equal(sc_x[b, :n].view(torch.int32), sc_y[b, :n].view(torch.int32)):
                return False
            for p in range(n):
                L = int(ln_x[b, p])
                if not (torch.equal(tok_x[b, p, :L], tok_y[b, p, :L]) and torch.equal(ts_x[b, p, :L], ts_y[b, p, :L])):
                    return False
        return True

    identical = same(outs["host"], outs["device"]) and same(outs["host"], outs["device+committed"])

    # the committed-prefix kernel beside an eos read-out (finalize) of the same states, CUDA events
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(labels, beam_width=Kb, device=dev, device_outputs=True)
    states = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    handles = (ctypes.c_void_p * B)(*[s.state for s in states])
    eos = (ctypes.c_uint8 * B)(*([1] * B))
    committed = torch.zeros(B, dtype=torch.int32, device=dev)
    c_tok = torch.empty(B, T, dtype=torch.int32, device=dev)
    c_ts = torch.empty(B, T, dtype=torch.int32, device=dev)
    f_tok = torch.empty(B, Kb, T, dtype=torch.int32, device=dev)
    f_ts = torch.empty(B, Kb, T, dtype=torch.int32, device=dev)
    f_sc = torch.empty(B, Kb, dtype=torch.float32, device=dev)
    f_ln = torch.empty(B, Kb, dtype=torch.int32, device=dev)
    f_nr = torch.empty(B, dtype=torch.int32, device=dev)
    f_fl = torch.empty(B, dtype=torch.int32, device=dev)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    kernel_ms, done = {}, 0
    for at in (100, 500, 1000):
        dec.decode(probs_d[:, done:at], states, [False] * B)
        done = at
        row = {}
        for name in ("committed", "finalize"):
            reps = []
            for _ in range(6):
                ev[0].record()
                if name == "committed":
                    _native.check(lib.ctcdec_stream_committed_device(handles, B, None, committed.data_ptr(),
                                                                     c_tok.data_ptr(), c_ts.data_ptr(), T, stream))
                else:  # a 0-frame chunk with every stream at eos: the per-call tables, then the finalize kernel
                    _native.check(lib.ctcdec_decode_stream_device(
                        probs_d.data_ptr(), -1, None, B, 0, handles, eos, f_tok.data_ptr(), f_ts.data_ptr(), T,
                        f_sc.data_ptr(), f_ln.data_ptr(), f_nr.data_ptr(), f_fl.data_ptr(), ws.data_ptr(), ws.numel(),
                        stream))
                ev[1].record()
                ev[1].synchronize()
                reps.append(ev[0].elapsed_time(ev[1]))
            row[name + "_ms"] = statistics.median(reps[1:])
        row["committed_depth_mean"] = float(committed.float().mean())
        kernel_ms["after_%d_frames" % at] = row
    for s in states:
        s.release()
    return {"workload": "config2 batch [256 x T=1000 x V=29], beam 100, OnlineCTCBeamDecoder", "chunk_frames": chunk,
            "card": card_info(local_rank), "paths": legs, "identical_final_outputs": bool(identical),
            "committed_vs_finalize": kernel_ms,
            "note": "per-chunk wall clock around the call; the device paths synchronise after every chunk, the host "
                    "path returns synchronised. committed_vs_finalize: CUDA events around one call of each entry "
                    "point, median of 5 after a warm-up call"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunk", type=int, default=16, help="frames per chunk call")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    torch.cuda.set_device(args.device)
    print(json.dumps(stream_leg(_native.load(), torch.device("cuda", args.device), args.device, args.chunk)), flush=True)


if __name__ == "__main__":
    main()
