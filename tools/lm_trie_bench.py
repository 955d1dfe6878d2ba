#!/usr/bin/env python
"""KenLM trie files in the device n-gram scorer: device memory, load time, upload time and the config-5-shaped call.

    python tools/lm_trie_bench.py --dir DIR [--lib NAME=PATH ...] [--reps N] [--rounds R]

DIR receives, when they are not there yet, a seeded word-based order-4 model generated with numpy (`large.arpa`:
--words words over the 29 labels' letters, more than 2^17 of them, and about 20 million n-grams) built by KenLM's
build_binary (oracle/_ref/build_binary, -S 1G -T DIR) as `probing`, `trie` and `-q 8 -b 8 -a 22 trie`, and the same
three types of the reference's test.arpa (config 5 as stated).

Each arm is one library (the in-tree build, or another build of the same ABI through CTCDECODE_B200_LIB: --lib
parent=build_variants/lib_parent.so) over one model file, run in a process of its own.  It reports the file's size,
ctcdec_scorer_table_bytes (when the library has it), the host load time (ctcdec_scorer_create_arpa), the first
decode's synchronised time and the median of --reps synchronised calls of the asynchronous entry
(ctcdec_decode_batch_lm_device_async) on config 5's shape ([64 x T=1000 x 29], beam 100, alpha 2.0, beta 1.0) timed
with CUDA events.  The large model decodes posteriors that spell sentences chained from its own 4-grams, so that its
lookups hit; test.arpa decodes config 5's text-driven batch.  Arms alternate: --rounds rounds of every (library,
model) pair.  Every arm of one model must give identical outputs (a hash of every result row).  The card, its power
limit and its clocks are read in the same run.  Prints one JSON line per arm, then a summary line.  Writes only DIR.
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BUILD_BINARY = os.path.join(ROOT, "oracle", "_ref", "build_binary")
TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
TYPES = {"probing": ["probing"], "trie": ["trie"], "qatrie": ["-q", "8", "-b", "8", "-a", "22", "trie"]}
LETTERS = "abcdefghijklmnopqrstuvwxyz'"


def generate(path, words=140000, counts=(8_000_000, 7_000_000, 5_000_000), seed=2027):
    """A seeded order-4 ARPA model.  Bigrams pair words with a Zipf-like skew; an n-gram of order 3 or 4 is an
    (n - 1)-gram context extended by a word that follows the context's last n - 2 words, so its context and its
    suffix are both in the model."""
    rng = np.random.default_rng(seed)
    spell = set()
    while len(spell) < words:
        n = rng.integers(3, 10, 4 * words)
        chars = rng.integers(0, 26, (4 * words, 9))
        for k in range(4 * words):
            spell.add("".join(LETTERS[c] for c in chars[k, :n[k]]))
            if len(spell) == words:
                break
    vocab = np.array(["<unk>", "<s>", "</s>"] + sorted(spell), dtype=object)
    V = len(vocab)
    zipf = 1.0 / np.arange(1, V - 2) ** 0.8
    zipf /= zipf.sum()

    def unique_rows(a):
        return np.unique(a, axis=0)
    grams = [None, None]
    a = 3 + rng.choice(V - 3, counts[0] * 6 // 5, p=zipf)
    b = 3 + rng.choice(V - 3, counts[0] * 6 // 5, p=zipf)
    a[: counts[0] // 50] = 1  # <s> w
    big = unique_rows(np.stack([a, b], 1))
    big = big[big[:, 0] != big[:, 1]]
    grams[1] = big[np.sort(rng.choice(len(big), min(len(big), counts[0]), replace=False))]
    for n in (3, 4):
        prev = grams[n - 2]
        # the (n - 1)-grams by their first n - 2 words: a context c extends by any w with c[1:] + (w,) in prev
        key = np.zeros(len(prev), np.int64)
        for k in range(n - 2):
            key = key * V + prev[:, k]
        order = np.argsort(key, kind="stable")
        skey = key[order]
        ckey = np.zeros(len(prev), np.int64)
        for k in range(1, n - 1):
            ckey = ckey * V + prev[:, k]
        lo = np.searchsorted(skey, ckey, "left")
        hi = np.searchsorted(skey, ckey, "right")
        has = np.nonzero(hi > lo)[0]
        pick = rng.choice(has, counts[n - 2] * 6 // 5)
        at = lo[pick] + (rng.random(len(pick)) * (hi[pick] - lo[pick])).astype(np.int64)
        new = np.concatenate([prev[pick], prev[order[at], n - 2:n - 1]], 1)
        new = unique_rows(new)
        grams.append(new[np.sort(rng.choice(len(new), min(len(new), counts[n - 2]), replace=False))])
    with open(path, "w") as f:
        f.write("\\data\\\nngram 1=%d\n" % V + "".join("ngram %d=%d\n" % (n, len(grams[n - 1])) for n in (2, 3, 4)))
        uni_p = -rng.uniform(1.0, 7.0, V).round(5)
        uni_p[1] = -99.0
        f.write("\n\\1-grams:\n")
        f.write("".join("%g\t%s\t%g\n" % (uni_p[i], vocab[i], -round(float(x), 5))
                        for i, x in enumerate(rng.uniform(0.0, 1.5, V))))
        for n in (2, 3, 4):
            g = grams[n - 1]
            f.write("\n\\%d-grams:\n" % n)
            probs = -rng.uniform(0.05, 5.0, len(g)).round(5)
            text = [" ".join(vocab[r]) for r in g]
            if n < 4:
                bos = -rng.uniform(0.0, 1.5, len(g)).round(5)
                f.write("".join("%g\t%s\t%g\n" % (p, t, b) for p, t, b in zip(probs, text, bos)))
            else:
                f.write("".join("%g\t%s\n" % (p, t) for p, t in zip(probs, text)))
        f.write("\n\\end\\\n")
    # sentences for the decode: 4-grams chained end to start where they can be, else simply concatenated
    pick = grams[3][rng.choice(len(grams[3]), 64 * 12)]
    texts = []
    for b in range(64):
        s = " ".join(" ".join(vocab[w] for w in row if w > 2) for row in pick[b * 12:(b + 1) * 12])
        texts.append(s[:250].rsplit(" ", 1)[0])
    return texts


def prepare(d):
    os.makedirs(d, exist_ok=True)
    arpa = os.path.join(d, "large.arpa")
    texts_path = os.path.join(d, "large.texts.json")
    if not os.path.exists(texts_path) and not os.path.exists(arpa):
        t0 = time.perf_counter()
        texts = generate(arpa)
        json.dump(texts, open(texts_path, "w"))
        print(json.dumps({"generated": arpa, "seconds": round(time.perf_counter() - t0, 1)}), flush=True)
    models = {}
    for name, src in (("large", arpa), ("test.arpa", TEST_ARPA)):
        for kind, args in TYPES.items():
            out = os.path.join(d, "%s.%s" % (name, kind))
            if not os.path.exists(out) and not os.path.exists(src):
                continue  # (DIR holds some of the large model's files without its ARPA source: those are run)
            if not os.path.exists(out):
                t0 = time.perf_counter()
                subprocess.run([BUILD_BINARY, "-S", "1G", "-T", d] + args + [src, out + ".tmp"], check=True,
                               stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
                os.replace(out + ".tmp", out)
                print(json.dumps({"built": out, "seconds": round(time.perf_counter() - t0, 1)}), flush=True)
            models["%s.%s" % (name, kind)] = out
    return models, texts_path


def arm(model, texts_path, reps):
    """one (library, model) arm in this process: JSON on stdout"""
    import torch
    from bench import CONFIGS, L29
    from ctcdecode_b200 import CTCBeamDecoder, _native
    from ctcdecode_b200.scorer import ArpaScorer
    from ctcdecode_b200.synth import text_probs
    from tests.test_lm import c5_text_probs
    cfg = CONFIGS["c5"]
    if os.path.basename(model).startswith("large."):
        probs = text_probs(json.load(open(texts_path)), L29, cfg["T"], seed=5)
    else:
        probs = c5_text_probs(cfg["B"], cfg["T"], seed=71)[0]
    x = probs.cuda()
    t0 = time.perf_counter()
    sc = ArpaScorer(L29, model, cfg["alpha"], cfg["beta"])
    load_s = time.perf_counter() - t0
    table = sc.table_bytes() if hasattr(_native.load(), "ctcdec_scorer_table_bytes") else None
    sc.release()
    dec = CTCBeamDecoder(L29, model_path=model, alpha=cfg["alpha"], beta=cfg["beta"], beam_width=cfg["beam"],
                         cutoff_top_n=cfg["cutoff_top_n"], cutoff_prob=cfg["cutoff_prob"], scorer_provider="device",
                         device_outputs=True, non_blocking=True)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    out = dec.decode(x)
    torch.cuda.synchronize()
    first_ms = 1e3 * (time.perf_counter() - t0)
    held = free0 - torch.cuda.mem_get_info()[0]
    dec.decode(x)
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = dec.decode(x)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    tok, sc_, ts, ln = [t.cpu() for t in out]
    nres, flags = dec.last_n_results.cpu(), dec.last_flags.cpu()
    h = hashlib.sha256(nres.numpy().tobytes() + flags.numpy().tobytes())
    for bb in range(nres.shape[0]):
        n = int(nres[bb])
        h.update(sc_[bb, :n].numpy().tobytes() + ln[bb, :n].numpy().tobytes())
        for p in range(n):
            L = int(ln[bb, p])
            h.update(tok[bb, p, :L].numpy().tobytes() + ts[bb, p, :L].numpy().tobytes())
    print(json.dumps({"model": os.path.basename(model), "file_bytes": os.path.getsize(model), "table_bytes": table,
                      "load_s": load_s, "first_call_ms": first_ms, "first_call_device_bytes": held,
                      "ms_median": statistics.median(ms), "ms_min": min(ms), "ms_max": max(ms), "calls": reps,
                      "outputs": h.hexdigest()}), flush=True)


def card():
    """name, power limit and clocks of GPU 0 (a read-only nvidia-smi query)"""
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", required=True)
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH: another build of the library, as an arm")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--arm", help=argparse.SUPPRESS)
    ap.add_argument("--texts", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.arm:
        return arm(args.arm, args.texts, args.reps)
    models, texts_path = prepare(args.dir)
    libs = [("tree", None)] + [tuple(s.split("=", 1)) for s in args.lib]
    results = {}
    before = card()
    for r in range(args.rounds):
        for name, model in models.items():
            for lib, path in libs:
                env = dict(os.environ)
                env.pop("CTCDECODE_B200_LIB", None)
                if path:
                    env["CTCDECODE_B200_LIB"] = os.path.abspath(path)
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--dir", args.dir, "--arm", model,
                                    "--texts", texts_path, "--reps", str(args.reps)], env=env, cwd=ROOT,
                                   capture_output=True, text=True)
                if p.returncode:
                    raise SystemExit("arm %s %s failed:\n%s" % (lib, name, p.stderr[-3000:]))
                rec = json.loads(p.stdout.strip().splitlines()[-1])
                rec.update(library=lib, round=r)
                print(json.dumps(rec), flush=True)
                results.setdefault(name, []).append(rec)
    same = {name: len({r["outputs"] for r in recs}) == 1 for name, recs in results.items()}
    summary = {}
    for name, recs in results.items():
        for lib, _ in libs:
            mine = [r for r in recs if r["library"] == lib]
            summary["%s %s" % (name, lib)] = {
                "ms_median_of_rounds": statistics.median(r["ms_median"] for r in mine),
                "load_s_median": statistics.median(r["load_s"] for r in mine),
                "first_call_ms_median": statistics.median(r["first_call_ms"] for r in mine),
                "table_bytes": mine[0]["table_bytes"], "file_bytes": mine[0]["file_bytes"]}
    print(json.dumps({"card_before": before, "card_after": card(), "summary": summary, "outputs_identical": same,
                      "note": "each arm a process of its own; CUDA events around each asynchronous call, synchronised "
                              "after it; arms alternate within each round"}), flush=True)
    assert all(same.values()), same


if __name__ == "__main__":
    main()
