"""The beam program with the library's own ARPA scorer computing its LM terms in the CTA (BeamParams::lm_dev), run in
the single-threaded CPU emulation (tests/native/emulate_ngram.cpp), against the reference build with its Scorer over
KenLM: tokens, timesteps, lens and float32 score bits equal."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, flat_probs, text_probs
from oracle import oracle as orc
from tests import golden_util
from tests.parity import compare

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]
TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran"]

needs_ref = pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)")
_i32p = ctypes.POINTER(ctypes.c_int32)
_f32p = ctypes.POINTER(ctypes.c_float)
_SRC = os.path.join(HERE, "native", "emulate_ngram.cpp")
_OUT = os.path.join(HERE, "native", "_build", "libctc_emul_ngram.so")
_lib = None


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
        _lib.emu_decode_batch_ngram.restype = ctypes.c_int
        _lib.emu_decode_batch_ngram.argtypes = [
            _f32p, _i32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int,
            ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_double, ctypes.c_double,
            ctypes.POINTER(ctypes.c_char_p), _i32p, _i32p, _f32p, _i32p, _i32p, _i32p]
    return _lib


def emu_decode(probs, labels, path, alpha, beta, seq_lens=None, beam=100, cutoff_prob=1.0, cutoff_top_n=40,
               blank_id=0, log_input=False, chunk=0):
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    B, T, V = probs.shape
    sl = None if seq_lens is None else np.ascontiguousarray(seq_lens, dtype=np.int32)
    tok = np.full((B, beam, T), -1, np.int32)
    ts = np.full((B, beam, T), -1, np.int32)
    sc = np.zeros((B, beam), np.float32)
    ln = np.zeros((B, beam), np.int32)
    nres = np.zeros((B,), np.int32)
    flags = np.zeros((B,), np.int32)
    lab = (ctypes.c_char_p * V)(*[x.encode() for x in labels])
    rc = _emu().emu_decode_batch_ngram(
        probs.ctypes.data_as(_f32p), sl.ctypes.data_as(_i32p) if sl is not None else None, B, T, V, beam, cutoff_prob,
        cutoff_top_n, blank_id, int(log_input), 0, chunk, path.encode(), alpha, beta, lab, tok.ctypes.data_as(_i32p),
        ts.ctypes.data_as(_i32p), sc.ctypes.data_as(_f32p), ln.ctypes.data_as(_i32p), nres.ctypes.data_as(_i32p),
        flags.ctypes.data_as(_i32p))
    assert rc == 0, rc
    return dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, n_results=nres, ties=flags)


@needs_ref
@pytest.mark.parametrize("chunk", [0, 7], ids=["one_launch", "chunks_of_7"])
@pytest.mark.parametrize("name", golden_util.names(lm=True) + golden_util.names_char())
def test_golden_fixtures(name, chunk):
    probs, seq_lens, kw, gold, alpha, beta = golden_util.load_lm(name)
    char = name.startswith("lmchar_")
    labels, path = (LCHAR, CHAR_LM) if char else (L29, TINY)
    got = emu_decode(probs, labels, path, alpha, beta, seq_lens=seq_lens, chunk=chunk, **kw)
    compare(gold, got, None, name)


@needs_ref
@pytest.mark.parametrize("order", ["0", "7"], ids=["thread_order_0", "thread_order_7"])
def test_config5_shape_on_test_arpa(order, monkeypatch):
    """BASELINE config 5's shape (beam 100, 29 labels, test.arpa, alpha 2.0, beta 1.0) at a length the emulation affords,
    under the forward and the reversed emulated thread orders"""
    monkeypatch.setenv("CTC_EMU_ORDER", order)
    probs = ctc_like_probs(2, 300, 29, seed=5).numpy()
    ref = orc.Reference(L29, model_path=TEST_ARPA, alpha=2.0, beta=1.0)
    want = ref.decode(probs, beam=100, num_processes=2)
    compare(want, emu_decode(probs, L29, TEST_ARPA, 2.0, 1.0, beam=100), None, "config 5 shape")


@needs_ref
@pytest.mark.parametrize("cfg", [
    dict(path="tiny", alpha=1.5, beta=0.8, beam=32, T=120, seed=11, seq_lens=[120, 0, 1, 57]),
    dict(path="tiny", alpha=2.0, beta=1.0, beam=16, T=100, seed=15, log_input=True),
    dict(path="test", alpha=1.0, beta=0.5, beam=48, T=90, seed=17, noise=True, cutoff_prob=0.99),
    dict(path="test", alpha=0.5, beta=-0.5, beam=30, T=80, seed=18, flat=True, cutoff_top_n=29),
    dict(path="char", alpha=1.0, beta=1.0, beam=20, T=70, seed=35, blank_id=5, cutoff_top_n=6),
    dict(path="char", alpha=2.5, beta=-1.0, beam=8, T=100, seed=33, log_input=True, seq_lens=[0, 1, 100]),
])
def test_against_live_reference(cfg):
    """ragged lengths with 0 and 1, log input, a blank other than 0, a top-n cut, a cutoff_prob cut and no cut"""
    cfg = dict(cfg)
    which, alpha, beta, T, seed = cfg.pop("path"), cfg.pop("alpha"), cfg.pop("beta"), cfg.pop("T"), cfg.pop("seed")
    path = dict(tiny=TINY, test=TEST_ARPA, char=CHAR_LM)[which]
    labels = LCHAR if which == "char" else L29
    seq_lens = cfg.pop("seq_lens", None)
    B = len(seq_lens) if seq_lens else 3
    if cfg.pop("noise", False) or which == "char":
        probs = ctc_like_probs(B, T, len(labels), seed=seed)
    elif cfg.pop("flat", False):
        probs = flat_probs(B, T, len(labels), seed=seed)
    else:
        probs = text_probs((TEXTS * 2)[:B], labels, T, seed=seed)
    if cfg.get("log_input"):
        probs = probs.log()
    probs = probs.numpy()
    sl = None if seq_lens is None else np.array(seq_lens, np.int32)
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    want = ref.decode(probs, sl, num_processes=2, **cfg)
    compare(want, emu_decode(probs, labels, path, alpha, beta, seq_lens=sl, **cfg), None, str(cfg))
