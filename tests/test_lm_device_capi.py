"""Argument checks and workspace size of the scorer path's device entry points (no GPU needed):
ctcdec_lm_workspace_bytes and ctcdec_decode_batch_lm_device.  The scorer is built through ctcdec_scorer_create with
dummy hooks, which are never called here.  (Decodes through the entry: tests/test_gpu_lm_device.py.)"""
import ctypes

import pytest
import torch

from ctcdecode_b200 import _native, build as libbuild

L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
_COND = ctypes.CFUNCTYPE(ctypes.c_double, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.c_int)(
    lambda c, l, n: -1.0)


@pytest.fixture(scope="module")
def lib():
    libbuild.build()
    return _native.load()


def _scorer(lib, labels, char_based=False):
    hooks = _native.ScorerHooks(None, ctypes.cast(_COND, ctypes.c_void_p).value, ctypes.cast(_COND, ctypes.c_void_p).value)
    lab = (ctypes.c_char_p * len(labels))(*[x.encode() for x in labels])
    words = ["the", "cat", "a"]
    wrd = (ctypes.c_char_p * len(words))(*[x.encode() for x in words])
    h = ctypes.c_void_p()
    assert lib.ctcdec_scorer_create(ctypes.byref(hooks), 1.0, 0.5, lab, len(labels), wrd, len(words), 3,
                                    1 if char_based else 0, ctypes.byref(h)) == 0
    return h


def _al256(x):
    return (x + 255) // 256 * 256


def _ws(lib, cfg, scorer, B, T):
    n = ctypes.c_size_t(0)
    rc = lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), scorer, B, T, ctypes.byref(n))
    return rc, n.value


@pytest.mark.parametrize("char_based", [False, True], ids=["word", "char"])
@pytest.mark.parametrize("shape", [(1, 1, 1), (3, 50, 16), (64, 1000, 100), (300, 20, 32), (5, 0, 8)])
def test_lm_workspace_is_the_plan_plus_the_lm_arrays(lib, char_based, shape):
    """the plan's regions (what ctcdec_workspace_bytes sizes: the layout a scorer changes is shared memory, not the
    workspace), then the per-node LM terms and dictionary states, the per-node rows of a character-based model and the
    device copy of seq_lens, each 256-byte aligned"""
    B, T, K = shape
    V = len(L29)
    sc = _scorer(lib, L29, char_based)
    try:
        cfg = _native.Config(V, K, 0, 0, 40, 1.0)
        plain = ctypes.c_size_t(0)
        assert lib.ctcdec_workspace_bytes(ctypes.byref(cfg), B, T, ctypes.byref(plain)) == 0
        nodes = B * (1 + K * T)
        want = (plain.value - 256) + 2 * _al256(nodes * 4) + (_al256(nodes * V * 4) if char_based else 0) \
            + _al256(B * 4) + 256
        assert _ws(lib, cfg, sc, B, T) == (0, want)
        assert lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), sc, B, T, None) == -1
    finally:
        lib.ctcdec_scorer_destroy(sc)


def test_lm_workspace_refusals(lib):
    sc = _scorer(lib, L29)
    ch = _scorer(lib, L29, char_based=True)
    try:
        # past the scorer's edge (704 at V = 29): the plan's message, which names the layout and the scorer
        assert _ws(lib, _native.Config(29, 704, 0, 0, 40, 1.0), sc, 8, 20)[0] == 0
        cfg = _native.Config(29, 705, 0, 0, 40, 1.0)
        plain = ctypes.c_size_t(0)
        assert lib.ctcdec_workspace_bytes(ctypes.byref(cfg), 8, 20, ctypes.byref(plain)) == 0  # (fits without one)
        assert _ws(lib, cfg, sc, 8, 20)[0] == -2
        msg = lib.ctcdec_last_error().decode()
        assert "with a scorer" in msg and "227 KB" in msg, msg
        # NULL scorer, and a scorer built for other labels
        assert _ws(lib, _native.Config(29, 16, 0, 0, 40, 1.0), None, 2, 10)[0] == -1
        assert b"scorer is NULL" in lib.ctcdec_last_error()
        assert _ws(lib, _native.Config(28, 16, 0, 0, 40, 1.0), sc, 2, 10)[0] == -1
        assert b"29 labels" in lib.ctcdec_last_error()
        # the rows of a character-based model beyond 64 GiB: 264 x (1 + 100 x 25000) x 29 x 4 bytes
        assert _ws(lib, _native.Config(29, 100, 0, 0, 40, 1.0), ch, 264, 25000)[0] == -2
        assert b"character-based" in lib.ctcdec_last_error()
        assert _ws(lib, _native.Config(29, 100, 0, 0, 40, 1.0), sc, 264, 25000)[0] == 0
    finally:
        lib.ctcdec_scorer_destroy(sc)
        lib.ctcdec_scorer_destroy(ch)


def _decode(lib, cfg, scorer, dtype=-1, B=2, T=10, outs=True, ws=0):
    buf = (ctypes.c_int32 * 64)()
    p = ctypes.addressof(buf) if outs else None   # (never dereferenced: every call here fails before)
    return lib.ctcdec_decode_batch_lm_device(ctypes.byref(cfg), scorer, p, dtype, None, B, T, p, p, p, p, p, p, None,
                                             p, ws, None)


def test_decode_lm_device_arguments(lib):
    """bad arguments are refused before any device is touched"""
    sc = _scorer(lib, L29)
    try:
        cfg = _native.Config(29, 16, 0, 0, 40, 1.0)
        assert _decode(lib, cfg, None) == -1
        assert b"scorer is NULL" in lib.ctcdec_last_error()
        assert _decode(lib, cfg, sc, dtype=7) == -1
        assert b"dtype 7" in lib.ctcdec_last_error()
        assert _decode(lib, _native.Config(30, 16, 0, 0, 40, 1.0), sc) == -1
        assert b"29 labels, decoder has 30" in lib.ctcdec_last_error()
        assert _decode(lib, cfg, sc, outs=False) == -1          # n_results / flags are required
        assert b"required" in lib.ctcdec_last_error()
        assert _decode(lib, _native.Config(29, 705, 0, 0, 40, 1.0), sc) == -2
        assert b"with a scorer" in lib.ctcdec_last_error()
        assert _decode(lib, cfg, sc, B=-1) == -1
    finally:
        lib.ctcdec_scorer_destroy(sc)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-device failure mode")
def test_decode_lm_device_without_gpu(lib):
    sc = _scorer(lib, L29)
    try:
        for dtype in (-1, 0, 1, 2):
            assert _decode(lib, _native.Config(29, 16, 0, 0, 40, 1.0), sc, dtype=dtype) == -5
            assert b"no CPU fallback" in lib.ctcdec_last_error()
    finally:
        lib.ctcdec_scorer_destroy(sc)
