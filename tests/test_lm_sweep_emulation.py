"""A sweep of the LM weights (ctcdec_decode_batch_lm_sweep_async) in the CPU emulation of the CTA program
(tests/native/emulate_sweep.cpp): P x B beam CTAs over one vocabulary scan, CTA g decoding input row g % B with its own
(alpha, beta) pair.  Every slice must equal the emulated single-pair decode at that pair (emulate_ngram_file.cpp), bit
for bit, and the reference build's decode after Scorer::reset_params with that pair."""
import ctypes
import os

import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, text_probs
from oracle import oracle as orc
from tests import tie_inputs
from tests.parity import compare
from tests.test_kenlm_binary import (BUILD_BINARY, CHAR_LM, L29, LCHAR, TEST_ARPA, TINY, _native_lib, build_binary,
                                     emu_decode)

needs_ref = pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)")
_i32p = ctypes.POINTER(ctypes.c_int32)
_f32p = ctypes.POINTER(ctypes.c_float)
_f64p = ctypes.POINTER(ctypes.c_double)
TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran", "a cat ran"]

# alpha = 0, beta < 0, and a beta large enough that the cutoff's max(0, beta) moves the cut
PAIRS_WORD = [(0.0, 0.0), (1.5, -0.8), (0.7, 4.0), (2.25, 1.1)]
PAIRS_CHAR = [(0.0, 1.0), (2.5, -1.0), (1.0, 3.5)]


def emu_sweep(probs, labels, path, pairs, seq_lens=None, beam=16, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0,
              log_input=False, nt=0):
    lib = _native_lib("emulate_sweep")
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    B, T, V = probs.shape
    P = len(pairs)
    sl = None if seq_lens is None else np.ascontiguousarray(seq_lens, dtype=np.int32)
    al = np.array([a for a, _ in pairs], np.float64)
    be = np.array([b for _, b in pairs], np.float64)
    tok, ts = np.full((P, B, beam, T), -1, np.int32), np.full((P, B, beam, T), -1, np.int32)
    sc, ln = np.zeros((P, B, beam), np.float32), np.zeros((P, B, beam), np.int32)
    nres, flags = np.zeros((P, B), np.int32), np.zeros((P, B), np.int32)
    lab = (ctypes.c_char_p * V)(*[x.encode() for x in labels])
    p = lambda a: a.ctypes.data_as(_i32p)  # noqa: E731
    rc = lib.emu_decode_sweep_ngram(
        probs.ctypes.data_as(_f32p), p(sl) if sl is not None else None, B, T, V, beam, ctypes.c_double(cutoff_prob),
        cutoff_top_n, blank_id, int(log_input), nt, path.encode(), al.ctypes.data_as(_f64p), be.ctypes.data_as(_f64p),
        P, lab, p(tok), p(ts), sc.ctypes.data_as(_f32p), p(ln), p(nres), p(flags))
    assert rc == 0, rc
    return dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, n_results=nres, ties=flags)


def _slice(d, p):
    return {k: v[p] for k, v in d.items()}


def _f32(x):
    return float(np.float32(x))


def check_sweep(probs, labels, path, pairs, ref_path=None, **kw):
    """every slice against the emulated single-pair decode (bit for bit, flags included) and the reference build"""
    got = emu_sweep(probs, labels, path, pairs, **kw)
    kw.pop("nt", None)
    ref = orc.Reference(labels, model_path=ref_path or path, alpha=1.0, beta=1.0) if orc.reference_available() else None
    sl = kw.pop("seq_lens", None)
    for p, (a, b) in enumerate(pairs):
        one = emu_decode(probs, labels, path, _f32(a), _f32(b), seq_lens=sl, **kw)
        s = _slice(got, p)
        for k in ("tokens", "timesteps", "lens", "n_results", "ties"):
            np.testing.assert_array_equal(s[k], one[k], err_msg="pair %d: %s" % (p, k))
        np.testing.assert_array_equal(s["scores"].view(np.uint32), one["scores"].view(np.uint32),
                                      err_msg="pair %d: score bits" % p)
        if ref is not None:
            ref.lib.ref_scorer_reset_params(ref.scorer, a, b)
            want = ref.decode(probs, sl, num_processes=2, **kw)
            compare(want, s, None, "pair %d (%g, %g)" % (p, a, b))
    return got


@needs_ref
def test_word_model_ragged_lengths():
    """tiny_lm, lengths T, 0, 1 and T / 2: the zero-length utterance has no frames in any pair"""
    probs = text_probs(TEXTS, L29, 60, seed=11).numpy()
    check_sweep(probs, L29, TINY, PAIRS_WORD, seq_lens=[60, 0, 1, 30], beam=16)


@needs_ref
def test_char_model_log_input_top_n():
    """char_lm (every label scored), log input, a blank other than 0 and a top-n cut"""
    probs = ctc_like_probs(3, 50, len(LCHAR), seed=35).log().numpy()
    check_sweep(probs, LCHAR, CHAR_LM, PAIRS_CHAR, seq_lens=[50, 0, 17], beam=12, cutoff_top_n=6, blank_id=5,
                log_input=True)


@needs_ref
def test_test_arpa_cutoff_prob():
    """test.arpa with a cutoff_prob cut"""
    probs = ctc_like_probs(2, 60, 29, seed=17).numpy()
    check_sweep(probs, L29, TEST_ARPA, PAIRS_WORD[:3], beam=24, cutoff_prob=0.99)


@needs_ref
def test_tie_prone_input_flags_every_pair():
    """quantised probabilities with a top-n cut: the scan's TIE_VOCAB bit shows in every pair's flags"""
    probs = tie_inputs.quantised_probs(3, 40, 29, seed=4)
    got = check_sweep(probs, L29, TINY, PAIRS_WORD[:3], beam=10, cutoff_top_n=8)
    vocab = got["ties"] & 4
    assert vocab[0].any(), "the input was meant to tie at the cut"
    for p in range(1, vocab.shape[0]):
        np.testing.assert_array_equal(vocab[p], vocab[0])


@needs_ref
def test_block_size_does_not_change_results():
    """the 128- and 256-thread programs give the same sweep on an input without comparator-equal results"""
    probs = text_probs(TEXTS[:3], L29, 50, seed=3).numpy()
    a = emu_sweep(probs, L29, TINY, PAIRS_WORD, beam=16, nt=128)
    b = emu_sweep(probs, L29, TINY, PAIRS_WORD, beam=16, nt=256)
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


@pytest.mark.skipif(not (orc.reference_available() and os.path.exists(BUILD_BINARY)),
                    reason="oracle/_ref (reference build and build_binary) not built")
def test_kenlm_trie_file(tmp_path):
    """a KenLM trie file of test.arpa sweeps to the same results as the ARPA text, and equals the reference over it"""
    trie = build_binary(TEST_ARPA, tmp_path, "trie")
    probs = ctc_like_probs(2, 50, 29, seed=21).numpy()
    got = check_sweep(probs, L29, trie, PAIRS_WORD[:3], beam=20, seq_lens=[50, 33])
    arpa = emu_sweep(probs, L29, TEST_ARPA, PAIRS_WORD[:3], beam=20, seq_lens=[50, 33])
    for k in got:
        np.testing.assert_array_equal(got[k], arpa[k], err_msg=k)
