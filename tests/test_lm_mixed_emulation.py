"""A decode over several language models (ctcdec_decode_batch_lm_mixed_async) in the CPU emulation of the CTA program
(tests/native/emulate_mixed.cpp): B beam CTAs, CTA b decoding with its own LM slot -- model, dictionary, order and
weights.  Every utterance must equal, bit for bit and flags included, the emulated single-model decode
(emulate_ngram_file.cpp) of the same batch with its model, under every emulated thread order."""
import ctypes
import os
import random

import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, text_probs
from tests.test_kenlm_binary import (BUILD_BINARY, CHAR_LM, L29, LCHAR, TEST_ARPA, TINY, _native_lib, build_binary,
                                     emu_decode)

_i32p = ctypes.POINTER(ctypes.c_int32)
_f32p = ctypes.POINTER(ctypes.c_float)
_f64p = ctypes.POINTER(ctypes.c_double)
TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran", "a cat ran", "the mat",
         "a dog sat"]
ORDERS = ["0", "1", "2"]   # CTC_EMU_ORDER: the order the emulation runs a region's threads in


def emu_mixed(probs, labels, models, lm_index, seq_lens=None, beam=16, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0,
              log_input=False, nt=0):
    """models: [(path, alpha, beta)]; utterance b decodes with models[lm_index[b]]"""
    lib = _native_lib("emulate_mixed")
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    B, T, V = probs.shape
    S = len(models)
    sl = None if seq_lens is None else np.ascontiguousarray(seq_lens, dtype=np.int32)
    idx = np.ascontiguousarray(lm_index, dtype=np.int32)
    paths = (ctypes.c_char_p * S)(*[m[0].encode() for m in models])
    al = np.array([m[1] for m in models], np.float64)
    be = np.array([m[2] for m in models], np.float64)
    tok, ts = np.full((B, beam, T), -1, np.int32), np.full((B, beam, T), -1, np.int32)
    sc, ln = np.zeros((B, beam), np.float32), np.zeros((B, beam), np.int32)
    nres, flags = np.zeros((B,), np.int32), np.zeros((B,), np.int32)
    lab = (ctypes.c_char_p * V)(*[x.encode() for x in labels])
    p = lambda a: a.ctypes.data_as(_i32p)  # noqa: E731
    rc = lib.emu_decode_mixed_ngram(
        probs.ctypes.data_as(_f32p), p(sl) if sl is not None else None, B, T, V, beam, ctypes.c_double(cutoff_prob),
        cutoff_top_n, blank_id, int(log_input), nt, paths, al.ctypes.data_as(_f64p), be.ctypes.data_as(_f64p), S,
        p(idx), lab, p(tok), p(ts), sc.ctypes.data_as(_f32p), p(ln), p(nres), p(flags))
    assert rc == 0, rc
    return dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, n_results=nres, ties=flags)


def check_mixed(monkeypatch, probs, labels, models, lm_index, seq_lens=None, **kw):
    """each utterance against the single-model emulation of the whole batch with its model, under every thread order"""
    for order in ORDERS:
        monkeypatch.setenv("CTC_EMU_ORDER", order)
        got = emu_mixed(probs, labels, models, lm_index, seq_lens=seq_lens, **kw)
        for s, (path, a, b) in enumerate(models):
            rows = [i for i, x in enumerate(lm_index) if x == s]
            if not rows:
                continue
            one = emu_decode(probs, labels, path, a, b, seq_lens=seq_lens, **kw)
            for k in ("tokens", "timesteps", "lens", "n_results", "ties"):
                np.testing.assert_array_equal(got[k][rows], one[k][rows], err_msg="order %s model %d: %s" % (order, s, k))
            np.testing.assert_array_equal(got["scores"][rows].view(np.uint32), one["scores"][rows].view(np.uint32),
                                          err_msg="order %s model %d: score bits" % (order, s))


WORD_MODELS = [(TEST_ARPA, 1.5, 0.8), (TEST_ARPA, 0.5, 2.0), (TINY, 2.0, -1.0)]


def test_word_models_ragged_uncut(monkeypatch):
    """test.arpa at two weight pairs and tiny_lm (orders 5 and 3), lengths T, 0, 1 and ragged, no vocabulary cut"""
    probs = text_probs(TEXTS, L29, 60, seed=11).numpy()
    check_mixed(monkeypatch, probs, L29, WORD_MODELS, [2, 0, 1, 0, 2, 1], seq_lens=[60, 0, 1, 45, 30, 60], beam=16,
                cutoff_top_n=40)


def test_word_models_cut_log_input(monkeypatch):
    """a top-8 cut of log-probabilities, and a model no utterance takes"""
    probs = np.log(ctc_like_probs(5, 50, 29, seed=7).numpy())
    check_mixed(monkeypatch, probs, L29, WORD_MODELS, [1, 1, 2, 1, 2], seq_lens=[50, 33, 0, 17, 50], beam=12,
                cutoff_top_n=8, log_input=True)


def _char_bigram(path, seed=5):
    """a second character-based model, of order 2, over char_lm.arpa's unigrams with other probabilities"""
    words = []
    with open(CHAR_LM, encoding="utf-8") as f:
        sect = None
        for line in f:
            line = line.rstrip("\n")
            if line.startswith("\\"):
                sect = line
                continue
            if sect == "\\1-grams:" and line.strip():
                words.append(line.split("\t")[1])
    rng = random.Random(seed)
    plain = [w for w in words if w not in ("<s>", "</s>", "<unk>")]
    bigrams = sorted({(rng.choice(["<s>"] + plain), rng.choice(plain + ["</s>"])) for _ in range(60)})
    with open(path, "w", encoding="utf-8") as f:
        f.write("\\data\\\nngram 1=%d\nngram 2=%d\n\n\\1-grams:\n" % (len(words), len(bigrams)))
        for w in words:
            lp = -99.0 if w == "<s>" else round(-0.4 - rng.random() * 1.6, 4)
            bo = "" if w == "</s>" else "\t%.4f" % (-0.1 - rng.random() * 0.5)
            f.write("%.4f\t%s%s\n" % (lp, w, bo))
        f.write("\n\\2-grams:\n")
        for a, b in bigrams:
            f.write("%.4f\t%s %s\n" % (-0.05 - rng.random() * 1.2, a, b))
        f.write("\n\\end\\\n")
    return path


def test_char_models(monkeypatch, tmp_path):
    """char_lm (order 3) beside a generated character bigram model: every label scored, per node rows of V terms"""
    other = _char_bigram(str(tmp_path / "char_bigram.arpa"))
    models = [(CHAR_LM, 1.0, 0.5), (other, 2.0, -0.5)]
    probs = ctc_like_probs(5, 40, len(LCHAR), seed=35).numpy()
    check_mixed(monkeypatch, probs, LCHAR, models, [1, 0, 1, 1, 0], seq_lens=[40, 0, 1, 23, 40], beam=10,
                cutoff_top_n=len(LCHAR))
    check_mixed(monkeypatch, probs, LCHAR, models, [0, 1, 0, 1, 1], beam=8, cutoff_top_n=6, blank_id=5)


@pytest.mark.skipif(not os.path.exists(BUILD_BINARY), reason="oracle/_ref build_binary not built")
def test_kenlm_trie_beside_arpa_text(monkeypatch, tmp_path):
    """a KenLM trie file of test.arpa beside tiny_lm's ARPA text"""
    trie = build_binary(TEST_ARPA, tmp_path, "trie")
    probs = ctc_like_probs(4, 40, 29, seed=21).numpy()
    check_mixed(monkeypatch, probs, L29, [(TINY, 1.0, 1.0), (trie, 1.5, 0.5)], [1, 0, 1, 1], seq_lens=[40, 31, 0, 40],
                beam=20)


def test_block_sizes_agree(monkeypatch):
    """the 128- and 256-thread programs give the same mixed decode on an input without comparator-equal results"""
    probs = text_probs(TEXTS[:4], L29, 50, seed=3).numpy()
    a = emu_mixed(probs, L29, WORD_MODELS, [0, 2, 1, 2], beam=16, nt=128)
    b = emu_mixed(probs, L29, WORD_MODELS, [0, 2, 1, 2], beam=16, nt=256)
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
