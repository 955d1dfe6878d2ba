"""Host-logic tests (no GPU) of the streaming arena compaction (ctcdecode_b200/csrc/compact_program.cuh), run by the
CPU emulation between the chunks of streaming decodes (tests/native/emulate_compact.cpp, emu_decode_stream_compact).

A stream compacted after any chunk, any number of times, must return what the same stream returns uncompacted, bit for
bit: the final rows, scores, lens, n_results and flags, and the committed prefix after every chunk.  Each compaction
must keep exactly the ancestors-or-self of the beam members, computed here from the arena dumped before it, renumbered
in the order of the old ids with parents, characters and jump pointers intact."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, flat_probs, text_probs
from tests import golden_util, tie_inputs
from tests.parity import compare

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]
TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran"]
_SRC = os.path.join(HERE, "native", "emulate_compact.cpp")
_OUT = os.path.join(HERE, "native", "_build", "libctc_emul_compact.so")
_i32p = ctypes.POINTER(ctypes.c_int32)
_f32p = ctypes.POINTER(ctypes.c_float)
_lib = None
_KJUMP = 16


def _emu():
    global _lib
    if _lib is None:
        os.makedirs(os.path.dirname(_OUT), exist_ok=True)
        csrc = os.path.join(ROOT, "ctcdecode_b200", "csrc")
        deps = [_SRC, os.path.join(HERE, "native", "emulate_cta.cpp")] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not (os.path.exists(_OUT) and all(os.path.getmtime(_OUT) >= os.path.getmtime(d) for d in deps)):
            tmp = _OUT + ".%d" % os.getpid()
            subprocess.run(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=off", "-fPIC", "-shared", "-nostdlib++",
                            "-Wno-unused-function", "-pthread", _SRC, "-o", tmp, "-l:libstdc++.so.6", "-lm"], check=True)
            os.replace(tmp, _OUT)
        _lib = ctypes.CDLL(_OUT)
        f = _lib.emu_decode_stream_compact
        f.restype = ctypes.c_int
        f.argtypes = [_f32p, _i32p] + [ctypes.c_int] * 4 + [ctypes.c_double] + [ctypes.c_int] * 4 + \
                     [_i32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_double,
                      ctypes.c_double, ctypes.POINTER(ctypes.c_char_p), _i32p, _i32p, _f32p, _i32p, _i32p, _i32p,
                      _i32p, _i32p, _i32p, _i32p, ctypes.c_longlong]
    return _lib


def _p(a, t):
    return a.ctypes.data_as(t)


def emu_stream(probs, chunks, every, seq_lens=None, beam=16, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0,
               log_input=False, slack=4, lm=None, labels=None, alpha=0.0, beta=0.0):
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    B, T, V = probs.shape
    sl = None if seq_lens is None else np.ascontiguousarray(seq_lens, dtype=np.int32)
    ch = np.ascontiguousarray(chunks, dtype=np.int32)
    nch, TT = len(ch), max(T, 1)
    out = dict(tokens=np.full((B, beam, T), -1, np.int32), timesteps=np.full((B, beam, T), -1, np.int32),
               scores=np.zeros((B, beam), np.float32), lens=np.zeros((B, beam), np.int32),
               n_results=np.zeros((B,), np.int32), ties=np.zeros((B,), np.int32),
               committed=np.zeros((nch, B), np.int32), com_tok=np.full((nch, B, TT), -7, np.int32),
               com_ts=np.full((nch, B, TT), -7, np.int32))
    dump = np.zeros(1 << 24, np.int32)
    lab = (ctypes.c_char_p * V)(*[x.encode() for x in labels]) if labels else None
    rc = _emu().emu_decode_stream_compact(
        _p(probs, _f32p), _p(sl, _i32p) if sl is not None else None, B, T, V, beam, cutoff_prob, cutoff_top_n,
        blank_id, int(log_input), 0, _p(ch, _i32p), nch, every, slack, lm.encode() if lm else None, alpha, beta, lab,
        _p(out["tokens"], _i32p), _p(out["timesteps"], _i32p), _p(out["scores"], _f32p), _p(out["lens"], _i32p),
        _p(out["n_results"], _i32p), _p(out["ties"], _i32p), _p(out["committed"], _i32p), _p(out["com_tok"], _i32p),
        _p(out["com_ts"], _i32p), _p(dump, _i32p), dump.size)
    assert rc == 0, rc
    out["compactions"] = _parse(dump)
    return out


def _parse(d):
    recs, i = [], 0
    while d[i] != -1:
        ci, b, n, M, A, kept = (int(x) for x in d[i:i + 6])
        i += 6
        r = dict(ci=ci, b=b, n=n, kept=kept)
        for k, m in (("par", n), ("chr", n), ("members", M), ("anchors", A), ("npar", kept), ("nchr", kept),
                     ("njump", kept)):
            r[k] = d[i:i + m].copy()
            i += m
        recs.append(r)
    return recs


def check_compaction(r):
    """The kept nodes are exactly the ancestors-or-self of the members, renumbered by old id."""
    par = r["par"]
    keep = np.zeros(r["n"], bool)
    for m in r["members"]:
        while m >= 0 and not keep[m]:
            keep[m] = True
            m = par[m]
    assert keep[0], "the root is an ancestor of every member"
    assert keep[r["anchors"]].all(), "an occupied dead anchor is not an ancestor of a member"
    assert r["kept"] == keep.sum(), "chunk %d stream %d: kept %d nodes, the members' closure has %d" % (
        r["ci"], r["b"], r["kept"], keep.sum())
    old = np.flatnonzero(keep)
    new_of = np.full(r["n"], -1, np.int64)
    new_of[old] = np.arange(len(old))
    npar = r["npar"]
    assert npar[0] == -1
    assert (npar[1:] >= 0).all() and (npar[1:] < np.arange(1, len(old))).all(), "a parent's id is not below its child's"
    assert np.array_equal(npar[1:], new_of[par[old[1:]]])
    assert np.array_equal(r["nchr"], r["chr"][old])
    depth = np.zeros(len(old), np.int64)
    for i in range(1, len(old)):
        depth[i] = depth[npar[i]] + 1
    assert r["njump"][0] == -1
    for i in range(1, len(old)):
        target, a = (depth[i] - 1) // _KJUMP * _KJUMP, i
        while depth[a] > target:
            a = npar[a]
        assert r["njump"][i] == a


_KEYS = ("tokens", "timesteps", "scores", "lens", "n_results", "ties", "committed", "com_tok", "com_ts")


def check(probs, chunks, everies=(1, 3), **kw):
    """Runs the stream never compacted and compacted every k-th chunk for each k; returns the never-compacted run."""
    base = emu_stream(probs, chunks, 0, **kw)
    assert base["compactions"] == []
    for every in everies:
        got = emu_stream(probs, chunks, every, **kw)
        assert len(got["compactions"]) == (len(chunks) // every) * probs.shape[0]
        for k in _KEYS:
            a, b = base[k], got[k]
            if a.dtype == np.float32:
                a, b = a.view(np.int32), b.view(np.int32)
            assert np.array_equal(a, b), "compaction every %d chunk(s) changed %s" % (every, k)
        for r in got["compactions"]:
            check_compaction(r)
        assert any(r["kept"] < r["n"] for r in got["compactions"]), "no compaction dropped a node"
    return base


def _oracle(cport, probs, base, seq_lens=None, **kw):
    kw = {k: v for k, v in kw.items() if k in ("beam", "cutoff_prob", "cutoff_top_n", "blank_id", "log_input")}
    ref = cport.decode_alternatives(probs, seq_lens, cap=256, **kw)
    compare(ref, {k: base[k] for k in ("tokens", "timesteps", "scores", "lens", "n_results", "ties")}, ref["ties"])


def _chunks(T, size):
    return [size] * -(-T // size)


@pytest.mark.parametrize("size", [1, 3, 17])
def test_chunk_sizes(cport, size):
    probs = ctc_like_probs(3, 60, 29, seed=40 + size).numpy()
    base = check(probs, _chunks(60, size), everies=(1, 4), beam=24)
    _oracle(cport, probs, base, beam=24)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_chunk_sizes(cport, seed):
    rng = np.random.RandomState(seed)
    T = 90
    chunks = []
    while sum(chunks) < T:
        chunks.append(int(rng.randint(1, 20)))
    probs = ctc_like_probs(3, T, 29, seed=50 + seed).numpy()
    base = check(probs, chunks, everies=(1, 2, 5), beam=20, seq_lens=[90, 61, 7])
    _oracle(cport, probs, base, beam=20, seq_lens=np.array([90, 61, 7], np.int32))


@pytest.mark.parametrize("cut", [dict(), dict(cutoff_top_n=10), dict(cutoff_prob=0.99)],
                         ids=["nothing_cut", "top_n", "cutoff_prob"])
def test_pruning_modes(cport, cut):
    probs = ctc_like_probs(3, 80, 29, seed=61).numpy()
    base = check(probs, _chunks(80, 7), beam=32, **cut)
    _oracle(cport, probs, base, beam=32, **cut)


def test_log_input_blank_last_ragged(cport):
    probs = ctc_like_probs(5, 70, 29, seed=62, blank_id=28, log=True).numpy()
    sl = [70, 33, 1, 0, 52]
    base = check(probs, _chunks(70, 9), beam=16, blank_id=28, log_input=True, seq_lens=sl)
    _oracle(cport, probs, base, beam=16, blank_id=28, log_input=True, seq_lens=np.array(sl, np.int32))


def test_beam_wider_than_the_live_trie(cport):
    # V = 3 at beam 64: the beam stays below its size, most of the trie stays alive
    probs = ctc_like_probs(3, 40, 3, seed=63).numpy()
    base = check(probs, _chunks(40, 6), beam=64)
    _oracle(cport, probs, base, beam=64)


@pytest.mark.parametrize("cfg", [dict(V=4, beam=8), dict(V=5, beam=3, blank_id=4),
                                 dict(V=6, beam=10, levels=(1.0, 2.0, 3.0, 5.0))])
def test_tie_prone_inputs(cfg):
    cfg = dict(cfg)
    V, levels = cfg.pop("V"), cfg.pop("levels", (1.0, 2.0, 4.0))
    probs = tie_inputs.quantised_probs(6, 30, V, seed=V + 10 * cfg["beam"], levels=levels)
    base = check(probs, _chunks(30, 4), **cfg)
    assert (base["ties"] & 1).any()  # the input does what it is for


@pytest.mark.parametrize("V,temp,seed", [(4, 1.0, 5), (3, 2.0, 2)])
def test_revival_heavy_inputs(cport, V, temp, seed):
    """tiny vocabularies and flat rows: dead anchors are revived through compacted arenas all the time"""
    probs = flat_probs(3, 200, V, seed, temp=temp).numpy()
    base = check(probs, _chunks(200, 5), everies=(1, 7), beam=16)
    _oracle(cport, probs, base, beam=16)


@pytest.mark.parametrize("order", range(8))
def test_emulated_thread_order(monkeypatch, order):
    """neither program's result may depend on the order the emulation runs its threads in"""
    monkeypatch.setenv("CTC_EMU_ORDER", str(order))
    probs = ctc_like_probs(3, 64, 29, seed=64).numpy()
    check(probs, _chunks(64, 5), everies=(1,), beam=40, seq_lens=[64, 50, 20])


@pytest.mark.parametrize("cfg", [
    dict(lm=TINY, alpha=1.5, beta=0.8, beam=32, T=90, seed=11, seq_lens=[90, 0, 1, 57]),
    dict(lm=TEST_ARPA, alpha=1.0, beta=0.5, beam=48, T=80, seed=17, noise=True, cutoff_prob=0.99),
    dict(lm=TEST_ARPA, alpha=-2.0, beta=1.0, beam=24, T=60, seed=18, cutoff_top_n=10),
    dict(lm=CHAR_LM, alpha=1.0, beta=1.0, beam=20, T=70, seed=35, blank_id=5, cutoff_top_n=6),
    dict(lm=CHAR_LM, alpha=2.5, beta=-1.0, beam=8, T=100, seed=33, log_input=True, seq_lens=[0, 1, 100]),
], ids=["tiny_ragged", "test_cutoff_prob", "test_negative_alpha", "char_top_n", "char_log_ragged"])
def test_device_ngram_scorer(cfg):
    cfg = dict(cfg)
    T, seed, sl = cfg.pop("T"), cfg.pop("seed"), cfg.pop("seq_lens", None)
    labels = LCHAR if cfg["lm"] == CHAR_LM else L29
    B = len(sl) if sl else 3
    if cfg.pop("noise", False) or cfg["lm"] == CHAR_LM:
        probs = ctc_like_probs(B, T, len(labels), seed=seed)
    else:
        probs = text_probs((TEXTS * 2)[:B], labels, T, seed=seed)
    if cfg.get("log_input"):
        probs = probs.log()
    check(probs.numpy(), _chunks(T, 7), labels=labels, seq_lens=sl, **cfg)


@pytest.mark.parametrize("name", [golden_util.names(lm=True)[0], golden_util.names_char()[0]])
def test_device_ngram_scorer_matches_reference_fixtures(name):
    probs, seq_lens, kw, gold, alpha, beta = golden_util.load_lm(name)
    char = name.startswith("lmchar_")
    labels, path = (LCHAR, CHAR_LM) if char else (L29, TINY)
    T = probs.shape[1]
    got = emu_stream(probs, _chunks(T, 7), 1, seq_lens=seq_lens, lm=path, labels=labels, alpha=alpha, beta=beta, **kw)
    for r in got["compactions"]:
        check_compaction(r)
    compare(gold, got, None, name)
