"""Argument checks and workspace size of the LM weight sweep (no GPU needed): ctcdec_lm_sweep_workspace_bytes and
ctcdec_decode_batch_lm_sweep_async refuse bad arguments before any device is touched.  (Decodes through the entry:
tests/test_gpu_lm_sweep.py.)"""
import ctypes
import os

import pytest
import torch

from ctcdecode_b200 import _native, build as libbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]
_COND = ctypes.CFUNCTYPE(ctypes.c_double, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.c_int)(
    lambda c, l, n: -1.0)


@pytest.fixture(scope="module")
def lib():
    libbuild.build()
    return _native.load()


def _arpa(lib, path, labels):
    lab = (ctypes.c_char_p * len(labels))(*[x.encode() for x in labels])
    h = ctypes.c_void_p()
    assert lib.ctcdec_scorer_create_arpa(path.encode(), 1.0, 0.5, lab, len(labels), ctypes.byref(h)) == 0
    return h


def _hook(lib, labels):
    hooks = _native.ScorerHooks(None, ctypes.cast(_COND, ctypes.c_void_p).value, ctypes.cast(_COND, ctypes.c_void_p).value)
    lab = (ctypes.c_char_p * len(labels))(*[x.encode() for x in labels])
    words = ["the", "cat", "a"]
    wrd = (ctypes.c_char_p * len(words))(*[x.encode() for x in words])
    h = ctypes.c_void_p()
    assert lib.ctcdec_scorer_create(ctypes.byref(hooks), 1.0, 0.5, lab, len(labels), wrd, len(words), 3, 0,
                                    ctypes.byref(h)) == 0
    return h


def _al256(x):
    return (x + 255) // 256 * 256


def _sweep_ws(lib, cfg, scorer, B, T, P):
    n = ctypes.c_size_t(0)
    rc = lib.ctcdec_lm_sweep_workspace_bytes(ctypes.byref(cfg), scorer, B, T, P, ctypes.byref(n))
    return rc, n.value


def _lm_ws(lib, cfg, scorer, B, T):
    n = ctypes.c_size_t(0)
    assert lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), scorer, B, T, ctypes.byref(n)) == 0
    return n.value


def _rows(n, T, V, top_n):
    """the pruned rows of n utterances: NP = the kept labels + 3 trailing floats, rounded up to 8; the cut's indices
    as well when the vocabulary is cut"""
    cut = top_n < V
    NP = ((min(V, top_n) if cut else V) + 3 + 7) // 8 * 8
    return _al256(n * T * NP * 4) + (_al256(n * T * NP * 2) if cut else 0)


@pytest.mark.parametrize("top_n", [40, 8], ids=["no_cut", "top8"])
@pytest.mark.parametrize("model", ["word", "char"])
@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (3, 50, 16, 4), (64, 1000, 100, 8), (5, 0, 8, 3), (300, 20, 32, 2)])
def test_sweep_workspace_is_the_documented_formula(lib, model, top_n, shape):
    """ctcdec_lm_workspace_bytes at P x B utterances, less the pruned rows of (P - 1) x B, plus the pairs' table"""
    B, T, K, P = shape
    path, labels = (TINY, L29) if model == "word" else (CHAR_LM, LCHAR)
    V = len(labels)
    sc = _arpa(lib, path, labels)
    try:
        cfg = _native.Config(V, K, 0, 0, top_n, 1.0)
        want = _lm_ws(lib, cfg, sc, P * B, T) - _rows(P * B, T, V, top_n) + _rows(B, T, V, top_n) + _al256(16 * P)
        assert _sweep_ws(lib, cfg, sc, B, T, P) == (0, want)
        if P == 1:
            assert want == _lm_ws(lib, cfg, sc, B, T) + 256
        assert lib.ctcdec_lm_sweep_workspace_bytes(ctypes.byref(cfg), sc, B, T, P, None) == -1
    finally:
        lib.ctcdec_scorer_destroy(sc)


def test_sweep_workspace_refusals(lib):
    sc = _arpa(lib, TINY, L29)
    ch = _arpa(lib, CHAR_LM, LCHAR)
    hk = _hook(lib, L29)
    try:
        cfg = _native.Config(29, 100, 0, 0, 40, 1.0)
        for P in (0, -1):
            assert _sweep_ws(lib, cfg, sc, 4, 10, P)[0] == -1
            assert b"at least one" in lib.ctcdec_last_error()
        assert _sweep_ws(lib, cfg, hk, 4, 10, 2)[0] == -2
        assert b"ctcdec_scorer_create_arpa" in lib.ctcdec_last_error()
        assert _sweep_ws(lib, cfg, None, 4, 10, 2)[0] == -1
        assert b"scorer is NULL" in lib.ctcdec_last_error()
        assert _sweep_ws(lib, _native.Config(28, 16, 0, 0, 40, 1.0), sc, 2, 10, 2)[0] == -1
        assert b"29 labels" in lib.ctcdec_last_error()
        assert _sweep_ws(lib, _native.Config(29, 705, 0, 0, 40, 1.0), sc, 2, 10, 2)[0] == -2
        assert b"with a scorer" in lib.ctcdec_last_error()
        # more beam CTAs than an int counts
        assert _sweep_ws(lib, cfg, sc, 1 << 12, 1, 1 << 20)[0] == -2
        assert b"too many beam CTAs" in lib.ctcdec_last_error()
        # the 64 GiB limits apply to the P x B utterances: histories of (1 + 100 x 1000) x 2 x 4 bytes each
        assert _sweep_ws(lib, cfg, sc, 64, 1000, 1000)[0] == 0
        assert _sweep_ws(lib, cfg, sc, 64, 1000, 1400)[0] == -2
        assert b"histories" in lib.ctcdec_last_error()
        # and the character-based model's rows: (1 + 100 x 1000) x 23 x 4 bytes each
        cc = _native.Config(len(LCHAR), 100, 0, 0, 40, 1.0)
        assert _sweep_ws(lib, cc, ch, 64, 1000, 8)[0] == 0
        assert _sweep_ws(lib, cc, ch, 64, 1000, 120)[0] == -2
        assert b"character-based" in lib.ctcdec_last_error()
    finally:
        for h in (sc, ch, hk):
            lib.ctcdec_scorer_destroy(h)


def _sweep(lib, cfg, scorer, alphas=(1.0, 2.0), betas=(0.5, 0.0), P=None, B=2, T=10, dtype=-1, outs=True):
    buf = (ctypes.c_int32 * 64)()
    p = ctypes.addressof(buf) if outs else None   # (never dereferenced: every call here fails before)
    P = len(alphas or betas) if P is None else P
    a = (ctypes.c_double * len(alphas))(*alphas) if alphas is not None else None
    b = (ctypes.c_double * len(betas))(*betas) if betas is not None else None
    return lib.ctcdec_decode_batch_lm_sweep_async(ctypes.byref(cfg), scorer, p, dtype, None, B, T, a, b, P, p, p, p,
                                                  p, p, p, None, p, 0, None)


def test_sweep_decode_arguments(lib):
    """bad arguments are refused before any device is touched"""
    sc = _arpa(lib, TINY, L29)
    hk = _hook(lib, L29)
    try:
        cfg = _native.Config(29, 16, 0, 0, 40, 1.0)
        assert _sweep(lib, cfg, sc, P=0) == -1
        assert b"at least one" in lib.ctcdec_last_error()
        assert _sweep(lib, cfg, hk) == -2
        assert b"ctcdec_scorer_create_arpa" in lib.ctcdec_last_error()
        assert _sweep(lib, cfg, None) == -1
        assert b"scorer is NULL" in lib.ctcdec_last_error()
        assert _sweep(lib, cfg, sc, alphas=None, P=2) == -1
        assert b"alphas and betas" in lib.ctcdec_last_error()
        assert _sweep(lib, cfg, sc, betas=None, P=2) == -1
        assert b"alphas and betas" in lib.ctcdec_last_error()
        assert _sweep(lib, cfg, sc, dtype=7) == -1
        assert b"dtype 7" in lib.ctcdec_last_error()
        assert _sweep(lib, cfg, sc, outs=False) == -1
        assert b"required" in lib.ctcdec_last_error()
        assert _sweep(lib, _native.Config(30, 16, 0, 0, 40, 1.0), sc) == -1
        assert b"29 labels, decoder has 30" in lib.ctcdec_last_error()
        assert _sweep(lib, cfg, sc, B=-1) == -1
    finally:
        lib.ctcdec_scorer_destroy(sc)
        lib.ctcdec_scorer_destroy(hk)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-device failure mode")
def test_sweep_decode_without_gpu(lib):
    sc = _arpa(lib, TINY, L29)
    try:
        for dtype in (-1, 0, 1, 2):
            assert _sweep(lib, _native.Config(29, 16, 0, 0, 40, 1.0), sc, dtype=dtype) == -5
            assert b"no CPU fallback" in lib.ctcdec_last_error()
    finally:
        lib.ctcdec_scorer_destroy(sc)
