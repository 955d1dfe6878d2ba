"""Argument checks and workspace size of a decode over several language models (no GPU needed):
ctcdec_lm_mixed_workspace_bytes and ctcdec_decode_batch_lm_mixed_async refuse bad arguments before any device is
touched.  (Decodes through the entry: tests/test_gpu_lm_mixed.py.)"""
import ctypes
import os

import pytest
import torch

from ctcdecode_b200 import _native, build as libbuild
from tests.test_lm_sweep_capi import CHAR_LM, L29, LCHAR, ROOT, TINY, _al256, _arpa, _hook, _lm_ws

TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")   # order 5 (tiny_lm: order 3)
MAX_MODELS = 16


@pytest.fixture(scope="module")
def lib():
    libbuild.build()
    return _native.load()


def _handles(scorers):
    return (ctypes.c_void_p * max(len(scorers), 1))(*[s.value if s is not None else None for s in scorers])


def _mixed_ws(lib, cfg, scorers, B, T, S=None):
    n = ctypes.c_size_t(0)
    S = len(scorers) if S is None else S
    rc = lib.ctcdec_lm_mixed_workspace_bytes(ctypes.byref(cfg), _handles(scorers), S, B, T, ctypes.byref(n))
    return rc, n.value


def _arena_stride(K, T):
    return 1 + K * T


@pytest.mark.parametrize("top_n", [40, 8], ids=["no_cut", "top8"])
@pytest.mark.parametrize("shape", [(1, 1, 1), (3, 50, 16), (64, 1000, 100), (5, 0, 8), (300, 20, 32)])
def test_mixed_workspace_is_the_documented_formula(lib, top_n, shape):
    """the workspace of the scorer of the largest order, plus the slot table (256 bytes a model) and the B slot
    indices; one scorer object given S times is ctcdec_lm_workspace_bytes"""
    B, T, K = shape
    tiny, tiny2, big = _arpa(lib, TINY, L29), _arpa(lib, TINY, L29), _arpa(lib, TEST_ARPA, L29)
    try:
        cfg = _native.Config(29, K, 0, 0, top_n, 1.0)
        for scorers in ([tiny, big], [big, tiny, tiny2], [tiny, tiny2]):
            rep = big if big in scorers else tiny
            want = _lm_ws(lib, cfg, rep, B, T) + _al256(256 * len(scorers)) + _al256(B)
            assert _mixed_ws(lib, cfg, scorers, B, T) == (0, want), scorers
        # the per-node histories take the largest order - 1 (4 ids for test.arpa, 2 for tiny_lm)
        hist = lambda n: _al256(B * _arena_stride(K, T) * n * 4)  # noqa: E731
        assert (_mixed_ws(lib, cfg, [tiny, big], B, T)[1] - _mixed_ws(lib, cfg, [tiny, tiny2], B, T)[1]
                == hist(4) - hist(2))
        for S in (1, 3):
            assert _mixed_ws(lib, cfg, [tiny] * S, B, T) == (0, _lm_ws(lib, cfg, tiny, B, T))
        assert lib.ctcdec_lm_mixed_workspace_bytes(ctypes.byref(cfg), _handles([tiny, big]), 2, B, T, None) == -1
    finally:
        for h in (tiny, tiny2, big):
            lib.ctcdec_scorer_destroy(h)


def test_character_models_workspace(lib):
    """two character-based models: the rows of V terms per node, as for one"""
    a, b = _arpa(lib, CHAR_LM, LCHAR), _arpa(lib, CHAR_LM, LCHAR)
    try:
        cfg = _native.Config(len(LCHAR), 12, 0, 0, 40, 1.0)
        assert _mixed_ws(lib, cfg, [a, b], 4, 30) == (0, _lm_ws(lib, cfg, a, 4, 30) + _al256(2 * 256) + _al256(4))
    finally:
        lib.ctcdec_scorer_destroy(a)
        lib.ctcdec_scorer_destroy(b)


def test_mixed_workspace_refusals(lib):
    tiny, big, ch, hk = _arpa(lib, TINY, L29), _arpa(lib, TEST_ARPA, L29), _arpa(lib, CHAR_LM, LCHAR), _hook(lib, L29)
    many = [_arpa(lib, TINY, L29) for _ in range(MAX_MODELS + 1)]
    try:
        cfg = _native.Config(29, 16, 0, 0, 40, 1.0)
        for S in (0, -1):
            assert _mixed_ws(lib, cfg, [tiny], 4, 10, S=S)[0] == -1
            assert b"a call takes 1 to 16" in lib.ctcdec_last_error()
        assert _mixed_ws(lib, cfg, many[:MAX_MODELS], 4, 10)[0] == 0
        assert _mixed_ws(lib, cfg, many, 4, 10)[0] == -1
        assert b"17 scorers" in lib.ctcdec_last_error()
        n = ctypes.c_size_t(0)
        assert lib.ctcdec_lm_mixed_workspace_bytes(ctypes.byref(cfg), None, 1, 4, 10, ctypes.byref(n)) == -1
        assert b"scorers is NULL" in lib.ctcdec_last_error()
        assert _mixed_ws(lib, cfg, [tiny, None], 4, 10)[0] == -1
        assert b"scorers[1] is NULL" in lib.ctcdec_last_error()
        # a hook scorer beside another scorer, either way round
        for pair in ([tiny, hk], [hk, big]):
            assert _mixed_ws(lib, cfg, pair, 4, 10)[0] == -2
            assert b"hook scorer" in lib.ctcdec_last_error()
        # word-based beside character-based
        assert _mixed_ws(lib, _native.Config(len(LCHAR), 16, 0, 0, 40, 1.0), [ch, tiny], 4, 10)[0] == -2
        assert b"both word-based or both character-based" in lib.ctcdec_last_error()
        # the decoder's labels, string for string
        other = list(L29)
        other[5] = "E"
        ot = _arpa(lib, TINY, other)
        try:
            assert _mixed_ws(lib, cfg, [tiny, ot], 4, 10)[0] == -1
            assert b"different labels" in lib.ctcdec_last_error()
        finally:
            lib.ctcdec_scorer_destroy(ot)
        assert _mixed_ws(lib, _native.Config(28, 16, 0, 0, 40, 1.0), [tiny, big], 2, 10)[0] == -1
        assert b"29 labels" in lib.ctcdec_last_error()
        assert _mixed_ws(lib, _native.Config(29, 705, 0, 0, 40, 1.0), [tiny, big], 2, 10)[0] == -2
        assert b"with a scorer" in lib.ctcdec_last_error()
    finally:
        for h in [tiny, big, ch, hk] + many:
            lib.ctcdec_scorer_destroy(h)


def _mixed(lib, cfg, scorers, lm_index, S=None, B=None, T=10, dtype=-1, outs=True):
    buf = (ctypes.c_int32 * 64)()
    p = ctypes.addressof(buf) if outs else None   # (never dereferenced: every call here fails before)
    S = len(scorers) if S is None else S
    B = len(lm_index) if B is None and lm_index is not None else (B or 0)
    idx = (ctypes.c_int32 * max(B, 1))(*lm_index) if lm_index is not None else None
    return lib.ctcdec_decode_batch_lm_mixed_async(ctypes.byref(cfg), _handles(scorers), S, idx, p, dtype, None, B, T,
                                                  p, p, p, p, p, p, None, p, 0, None)


def test_mixed_decode_arguments(lib):
    """bad arguments are refused before any device is touched"""
    tiny, big, ch, hk = _arpa(lib, TINY, L29), _arpa(lib, TEST_ARPA, L29), _arpa(lib, CHAR_LM, LCHAR), _hook(lib, L29)
    try:
        cfg = _native.Config(29, 16, 0, 0, 40, 1.0)
        assert _mixed(lib, cfg, [tiny, big], [0, 1], S=0) == -1
        assert b"a call takes 1 to 16" in lib.ctcdec_last_error()
        assert _mixed(lib, cfg, [tiny, big], [0, 2]) == -1
        assert b"lm_index[1] = 2 outside [0, 2)" in lib.ctcdec_last_error()
        assert _mixed(lib, cfg, [tiny, big], [-1, 0]) == -1
        assert b"lm_index[0] = -1" in lib.ctcdec_last_error()
        assert _mixed(lib, cfg, [tiny, big], None, B=2) == -1
        assert b"lm_index (host int32[B]) is NULL" in lib.ctcdec_last_error()
        assert _mixed(lib, cfg, [tiny, hk], [0, 1]) == -2
        assert b"hook scorer" in lib.ctcdec_last_error()
        # one hook scorer alone is the single-model asynchronous call, which takes none
        assert _mixed(lib, cfg, [hk, hk], [0, 1]) == -2
        assert b"ctcdec_scorer_create_arpa" in lib.ctcdec_last_error()
        assert _mixed(lib, _native.Config(len(LCHAR), 16, 0, 0, 40, 1.0), [ch, tiny], [0, 1]) == -2
        assert b"both word-based or both character-based" in lib.ctcdec_last_error()
        assert _mixed(lib, cfg, [tiny, big], [0, 1], dtype=7) == -1
        assert b"dtype 7" in lib.ctcdec_last_error()
        assert _mixed(lib, cfg, [tiny, big], [0, 1], outs=False) == -1
        assert b"required" in lib.ctcdec_last_error()
        assert _mixed(lib, _native.Config(30, 16, 0, 0, 40, 1.0), [tiny, big], [0, 1]) == -1
        assert b"29 labels, decoder has 30" in lib.ctcdec_last_error()
    finally:
        for h in (tiny, big, ch, hk):
            lib.ctcdec_scorer_destroy(h)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-device failure mode")
def test_mixed_decode_without_gpu(lib):
    tiny, big = _arpa(lib, TINY, L29), _arpa(lib, TEST_ARPA, L29)
    try:
        for dtype in (-1, 0, 1, 2):
            assert _mixed(lib, _native.Config(29, 16, 0, 0, 40, 1.0), [tiny, big], [1, 0], dtype=dtype) == -5
            assert b"no CPU fallback" in lib.ctcdec_last_error()
    finally:
        lib.ctcdec_scorer_destroy(tiny)
        lib.ctcdec_scorer_destroy(big)
