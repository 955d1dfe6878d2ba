"""Host-logic tests (no GPU) of the committed-prefix program (committed_cta_run in
ctcdecode_b200/csrc/beam_program.cuh), run by the CPU emulation after every chunk of a streaming decode
(tests/native/emulate_committed.cpp, emu_decode_stream_committed).

After every chunk the committed prefix -- the path from the trie root to the lowest common ancestor of the beam
members -- must be the longest common prefix (tokens and timesteps) of the rows the C oracle returns for the frames
consumed so far, or of one of the outputs the reference may produce where the oracle flags a beam-cut tie.  It never
shrinks, reading it in deltas (since = the previous depth) gives the same path, an invalid `since` reads it from 0,
and the final prefix starts every row of the stream's final output."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, flat_probs
from tests import tie_inputs
from tests.parity import compare

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "native", "emulate_committed.cpp")
_OUT = os.path.join(_HERE, "native", "_build", "libctc_emul_committed.so")
_i32p = ctypes.POINTER(ctypes.c_int32)
_f32p = ctypes.POINTER(ctypes.c_float)
_lib = None


def _build():
    """Compiles tests/native/emulate_committed.cpp (which includes emulate_cta.cpp) like tests/emul.py does."""
    global _lib
    if _lib is None:
        os.makedirs(os.path.dirname(_OUT), exist_ok=True)
        csrc = os.path.join(_HERE, "..", "ctcdecode_b200", "csrc")
        deps = [_SRC, os.path.join(_HERE, "native", "emulate_cta.cpp")] + \
            [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not (os.path.exists(_OUT) and all(os.path.getmtime(_OUT) >= os.path.getmtime(d) for d in deps)):
            tmp = _OUT + ".tmp%d" % os.getpid()
            subprocess.run(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=off", "-fPIC", "-shared",
                            "-nostdlib++", "-Wno-unused-function", "-pthread", _SRC, "-o", tmp, "-l:libstdc++.so.6",
                            "-lm"], check=True)
            os.replace(tmp, _OUT)
        _lib = ctypes.CDLL(_OUT)
    return _lib


def _p(a, t):
    return a.ctypes.data_as(t)


def emu_stream_committed(probs, seq_lens, chunk, beam, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0,
                         log_input=False, nt=0):
    lib = _build()
    f = lib.emu_decode_stream_committed
    f.restype = ctypes.c_int
    f.argtypes = [_f32p, _i32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                  ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int] + [_i32p, _i32p, _f32p] + \
                 [_i32p] * 10
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    B, T, V = probs.shape
    sl = None if seq_lens is None else np.ascontiguousarray(seq_lens, dtype=np.int32)
    nch = max(1, -(-T // chunk))
    out = dict(tokens=np.full((B, beam, T), -1, np.int32), timesteps=np.full((B, beam, T), -1, np.int32),
               scores=np.zeros((B, beam), np.float32), lens=np.zeros((B, beam), np.int32),
               n_results=np.zeros((B,), np.int32), ties=np.zeros((B,), np.int32),
               committed=np.zeros((nch, B), np.int32))
    for k in ("full", "acc", "bad"):
        out[k + "_tok"] = np.full((nch, B, max(T, 1)), -7, np.int32)
        out[k + "_ts"] = np.full((nch, B, max(T, 1)), -7, np.int32)
    rc = f(_p(probs, _f32p), _p(sl, _i32p) if sl is not None else None, B, T, V, beam, cutoff_prob, cutoff_top_n,
           blank_id, int(log_input), nt, chunk, _p(out["tokens"], _i32p), _p(out["timesteps"], _i32p),
           _p(out["scores"], _f32p), _p(out["lens"], _i32p), _p(out["n_results"], _i32p), _p(out["ties"], _i32p),
           _p(out["committed"], _i32p), _p(out["full_tok"], _i32p), _p(out["full_ts"], _i32p),
           _p(out["acc_tok"], _i32p), _p(out["acc_ts"], _i32p), _p(out["bad_tok"], _i32p), _p(out["bad_ts"], _i32p))
    assert rc == 0, rc
    return out


def lcp(d, b):
    """(depth, tokens, timesteps) of the longest common prefix of the n_results rows of utterance b."""
    n = int(d["n_results"][b])
    if n == 0:
        return 0, np.zeros(0, np.int32), np.zeros(0, np.int32)
    L0 = int(d["lens"][b, 0])
    t0, s0 = d["tokens"][b, 0, :L0], d["timesteps"][b, 0, :L0]
    D = L0
    for p in range(1, n):
        L = min(D, int(d["lens"][b, p]))
        same = (d["tokens"][b, p, :L] == t0[:L]) & (d["timesteps"][b, p, :L] == s0[:L])
        D = L if same.all() else int(np.argmin(same))
    return D, t0[:D], s0[:D]


def check_stream(cport, probs, seq_lens, chunk, **kw):
    """Runs the emulation and checks the committed prefix after every chunk against the oracle.  Returns the number
    of (chunk, stream) points compared with the oracle and how many were skipped as unresolved (junk ties)."""
    B, T, V = probs.shape
    lens = np.full(B, T, np.int64) if seq_lens is None else np.clip(np.asarray(seq_lens, np.int64), 0, T)
    got = emu_stream_committed(probs, seq_lens, chunk, **kw)
    nch = got["committed"].shape[0]
    checked = unresolved = 0
    prev = np.zeros(B, np.int64)
    for ci in range(nch):
        tc = min(T, (ci + 1) * chunk)
        consumed = np.minimum(lens, tc).astype(np.int32)
        ref = cport.decode_alternatives(probs[:, :tc], consumed, cap=256, **kw)
        for b in range(B):
            D = int(got["committed"][ci, b])
            assert D >= 0, "chunk %d stream %d: the three committed calls disagree" % (ci, b)
            assert D >= prev[b], "chunk %d stream %d: committed depth shrank %d -> %d" % (ci, b, prev[b], D)
            assert D <= consumed[b]
            prev[b] = D
            ft, fs = got["full_tok"][ci, b, :D], got["full_ts"][ci, b, :D]
            assert np.array_equal(got["acc_tok"][ci, b, :D], ft) and np.array_equal(got["acc_ts"][ci, b, :D], fs), \
                "chunk %d stream %d: deltas do not add up to the whole prefix" % (ci, b)
            assert np.array_equal(got["bad_tok"][ci, b, :D], ft) and np.array_equal(got["bad_ts"][ci, b, :D], fs)
            if D < T:  # nothing beyond the prefix is written
                assert (got["full_tok"][ci, b, D:] == -7).all()
            if ref["unresolved"][b]:
                unresolved += 1
                continue
            ok = False
            for alt in ref["alternatives"][b]:
                Dr, rt, rs = lcp(alt, 0)
                if Dr == D and np.array_equal(rt, ft) and np.array_equal(rs, fs):
                    ok = True
                    break
            assert ok, "chunk %d stream %d: committed prefix (depth %d) is not the common prefix of the reference's " \
                       "rows (depth %d)" % (ci, b, D, lcp(ref, b)[0])
            checked += 1
    # the final decode is the oracle's, and the last committed prefix starts each of its rows
    ref = cport.decode_alternatives(probs, seq_lens, cap=256, **kw)
    compare(ref, {k: got[k] for k in ("tokens", "timesteps", "scores", "lens", "n_results", "ties")}, ref["ties"])
    for b in range(B):
        D = int(got["committed"][-1, b])
        for p in range(int(got["n_results"][b])):
            assert np.array_equal(got["tokens"][b, p, :D], got["full_tok"][-1, b, :D])
            assert np.array_equal(got["timesteps"][b, p, :D], got["full_ts"][-1, b, :D])
    return checked, unresolved, got


@pytest.mark.parametrize("chunk", [7, 16])
def test_committed_config2_shape(cport, chunk):
    probs = ctc_like_probs(3, 64, 29, seed=31).numpy()
    checked, unresolved, got = check_stream(cport, probs, None, chunk, beam=100)
    assert unresolved == 0 and checked == 3 * -(-64 // chunk)


def test_committed_config4_shape(cport):
    probs = ctc_like_probs(1, 120, 256, seed=32).numpy()
    checked, unresolved, _ = check_stream(cport, probs, None, 20, beam=200, cutoff_prob=0.99)
    assert unresolved == 0


@pytest.mark.parametrize("cfg", [
    dict(V=4, beam=8),
    dict(V=5, beam=3, blank_id=4),
    dict(V=6, beam=10, levels=(1.0, 2.0, 3.0, 5.0)),
])
def test_committed_tie_prone_inputs(cport, cfg):
    cfg = dict(cfg)
    V, levels = cfg.pop("V"), cfg.pop("levels", (1.0, 2.0, 4.0))
    probs = tie_inputs.quantised_probs(6, 24, V, seed=V + 10 * cfg["beam"], levels=levels)
    checked, unresolved, got = check_stream(cport, probs, None, 5, **cfg)
    assert (got["ties"] & 1).any()  # the input does what it is for
    assert checked >= 20


def test_committed_flat_rows(cport):
    probs = flat_probs(3, 60, 5, seed=3, temp=2.0).numpy()
    check_stream(cport, probs, None, 9, beam=16)


def test_committed_beam1_is_the_best_path(cport):
    probs = ctc_like_probs(3, 70, 29, seed=33).numpy()
    _, _, got = check_stream(cport, probs, [70, 33, 1], 8, beam=1)
    assert np.array_equal(got["committed"][-1], got["lens"][:, 0])


def test_committed_beam_not_full_and_empty_streams(cport):
    # V = 3 and beam 64: the beam stays below its size for many frames; streams of 0 frames commit nothing
    probs = ctc_like_probs(4, 40, 3, seed=34).numpy()
    _, _, got = check_stream(cport, probs, [40, 0, 13, 0], 6, beam=64)
    assert (got["n_results"] < 64).any()
    assert (got["committed"][:, 1] == 0).all() and (got["committed"][:, 3] == 0).all()


def test_committed_ragged_lengths(cport):
    probs = ctc_like_probs(5, 90, 29, seed=35).numpy()
    check_stream(cport, probs, [90, 45, 3, 1, 77], 11, beam=24, cutoff_top_n=10)


@pytest.mark.parametrize("order", [1, 3, 7])
def test_committed_emulated_thread_order(cport, monkeypatch, order):
    """The program's result must not depend on the order the emulation runs its threads in."""
    monkeypatch.setenv("CTC_EMU_ORDER", str(order))
    probs = ctc_like_probs(3, 64, 29, seed=36).numpy()
    check_stream(cport, probs, [64, 50, 20], 10, beam=32)
