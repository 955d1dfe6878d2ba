"""The scorer path at every language-model weight the scorers accept, in the CPU emulation of the CTA program, against
the reference build: tokens, timesteps, lens and float32 score bits equal.

With a scorer the beam kernel selects each frame's top K through a radix histogram laid over the score keys
[lo32, top32].  A scored candidate's LM term float(cond_log_prob * alpha) is positive when alpha < 0, or when a positive
backoff weight lifts a conditional log-prob above 0, so top32 has to bound the terms a frame can add, not assume them
<= 0.  The emulation stops a decode whose key lands outside the histogram (CTC_HIST_ADD in beam_program.cuh), so these
cases fail loudly if the range misses a key."""
import os

import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, flat_probs, text_probs
from oracle import oracle as orc
from tests import emul
from tests.parity import compare
from tests.test_kenlm_binary import BUILD_BINARY, build_binary
from tests.test_kenlm_binary import emu_decode as emu_decode_file
from tests.test_lm_sweep_emulation import check_sweep
from tests.test_ngram_emulation import CHAR_LM, L29, LCHAR, TEST_ARPA, TINY, emu_decode

needs_ref = pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref (the reference build) not built")
PATHS = dict(tiny=TINY, test=TEST_ARPA, char=CHAR_LM)
TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran"]

# A word model whose backoff weights are positive: a backed-off conditional log-prob backoff(h) + p(w) is above 0, e.g.
# p(sat | the) = 0.8 - 0.7 and p(cat | <s>) = 1.2 - 0.5 (log10).  KenLM and the library's loader both accept it.
POSITIVE_BACKOFF_ARPA = """\\data\\
ngram 1=7
ngram 2=4

\\1-grams:
-1.0\t<unk>\t0
-99\t<s>\t1.2
-0.6\t</s>
-0.4\tthe\t0.8
-0.5\tcat\t1.0
-0.7\tsat\t0.5
-0.9\ton\t0.3

\\2-grams:
-0.3\t<s> the
-0.2\tthe cat
-0.4\tcat sat
-0.6\tsat on

\\end\\
"""
BACKOFF_TEXTS = ["the cat sat on the cat", "cat sat the on", "on the sat cat sat"]


def _probs(which, B, T, V, seed, kind):
    if kind == "text":
        return text_probs((TEXTS * 2)[:B], L29, T, seed=seed)
    if kind == "flat":
        return flat_probs(B, T, V, seed=seed)
    return ctc_like_probs(B, T, V, seed=seed)


# every alpha in {-5, -2, -0.5, 0} and every beta in {-4, 0, 1, 4, 10} at least once, on the three models; top-n and
# cutoff_prob cuts and no cut, log input, ragged lengths with 0 and 1, and launches of 7 frames (the streaming shape)
DEVICE_CASES = [
    dict(path="test", alpha=-2.0, beta=1.0, beam=32, T=120, B=2, seed=5),
    dict(path="test", alpha=-5.0, beta=0.0, beam=32, T=120, B=2, seed=5),
    dict(path="test", alpha=-0.5, beta=-4.0, beam=48, T=90, B=3, seed=17, cutoff_prob=0.99),
    dict(path="test", alpha=0.0, beta=4.0, beam=30, T=80, B=3, seed=18, kind="flat", cutoff_top_n=20),
    dict(path="test", alpha=-2.0, beta=10.0, beam=24, T=100, B=2, seed=19, chunk=7),
    dict(path="tiny", alpha=-2.0, beta=1.0, beam=32, T=120, B=3, seed=11, kind="text", seq_lens=[120, 0, 1]),
    dict(path="tiny", alpha=-5.0, beta=10.0, beam=16, T=100, B=3, seed=15, kind="text", log_input=True),
    dict(path="tiny", alpha=-0.5, beta=0.0, beam=20, T=100, B=2, seed=16, kind="text", cutoff_top_n=8, chunk=7),
    dict(path="char", alpha=-0.5, beta=0.0, beam=16, T=40, B=1, seed=5),
    dict(path="char", alpha=-2.0, beta=1.0, beam=20, T=70, B=3, seed=35, blank_id=5, cutoff_top_n=6),
    dict(path="char", alpha=-5.0, beta=4.0, beam=8, T=100, B=3, seed=33, log_input=True, seq_lens=[0, 1, 100]),
    dict(path="char", alpha=-2.0, beta=-4.0, beam=24, T=80, B=2, seed=34, cutoff_prob=0.95, chunk=7),
    dict(path="char", alpha=0.0, beta=10.0, beam=12, T=60, B=2, seed=36, kind="flat"),
]


def _case_id(cfg):
    return "%s_a%g_b%g_k%d%s" % (cfg["path"], cfg["alpha"], cfg["beta"], cfg["beam"],
                                 "_chunk%d" % cfg["chunk"] if cfg.get("chunk") else "")


def _inputs(cfg):
    cfg = dict(cfg)
    which = cfg.pop("path")
    labels = LCHAR if which == "char" else L29
    probs = _probs(which, cfg.pop("B"), cfg.pop("T"), len(labels), cfg.pop("seed"), cfg.pop("kind", "noise"))
    if cfg.get("log_input"):
        probs = probs.log()
    sl = cfg.pop("seq_lens", None)
    return which, labels, probs.numpy(), None if sl is None else np.array(sl, np.int32), cfg


@needs_ref
@pytest.mark.parametrize("cfg", DEVICE_CASES, ids=[_case_id(c) for c in DEVICE_CASES])
def test_device_scorer(cfg):
    which, labels, probs, sl, kw = _inputs(cfg)
    alpha, beta, chunk = kw.pop("alpha"), kw.pop("beta"), kw.pop("chunk", 0)
    ref = orc.Reference(labels, model_path=PATHS[which], alpha=alpha, beta=beta)
    want = ref.decode(probs, sl, num_processes=2, **kw)
    got = emu_decode(probs, labels, PATHS[which], alpha, beta, seq_lens=sl, chunk=chunk, **kw)
    compare(want, got, None, _case_id(cfg))


@pytest.fixture
def backoff_arpa(tmp_path):
    path = tmp_path / "positive_backoff.arpa"
    path.write_text(POSITIVE_BACKOFF_ARPA)
    return str(path)


def _cond(ref, text):
    """the reference Scorer's conditional log-prob of the last word of `text` (not weighted by alpha)"""
    ids = np.array([L29.index(ch) for ch in text], np.int32)
    return ref.lib.ref_scorer_cond_from_labels(ref.scorer, ids.ctypes.data_as(emul._i32p), len(ids))


@needs_ref
@pytest.mark.parametrize("chunk", [0, 7], ids=["one_launch", "chunks_of_7"])
def test_positive_backoff_model(backoff_arpa, chunk):
    """alpha = 1.5 > 0, yet the LM terms of backed-off words are positive"""
    ref = orc.Reference(L29, model_path=backoff_arpa, alpha=1.5, beta=0.5)
    assert _cond(ref, "the sat") > 0 and _cond(ref, "cat") > 0, "the model was meant to have positive conditionals"
    probs = text_probs(BACKOFF_TEXTS, L29, 120, seed=41).numpy()
    want = ref.decode(probs, beam=32, num_processes=2)
    compare(want, emu_decode(probs, L29, backoff_arpa, 1.5, 0.5, beam=32, chunk=chunk), None, "positive backoff")


@pytest.mark.skipif(not (orc.reference_available() and os.path.exists(BUILD_BINARY)),
                    reason="oracle/_ref (reference build and build_binary) not built")
def test_positive_backoff_model_as_kenlm_trie(backoff_arpa, tmp_path):
    """the same model as a KenLM trie file, searched in place by the device scorer"""
    trie = build_binary(backoff_arpa, tmp_path, "trie")
    ref = orc.Reference(L29, model_path=trie, alpha=1.5, beta=0.5)
    assert _cond(ref, "the sat") > 0
    probs = ctc_like_probs(3, 100, 29, seed=42).numpy()
    sl = np.array([100, 1, 64], np.int32)
    want = ref.decode(probs, sl, beam=24, num_processes=2)
    compare(want, emu_decode_file(probs, L29, trie, 1.5, 0.5, seq_lens=sl, beam=24), None, "positive backoff, trie")


HOOK_CASES = [
    dict(path="tiny", alpha=-2.0, beta=1.0, beam=32, T=100, B=3, seed=12, kind="text"),
    dict(path="test", alpha=-5.0, beta=0.0, beam=24, T=80, B=2, seed=5, chunk=7),
    dict(path="char", alpha=-2.0, beta=1.0, beam=16, T=60, B=2, seed=31),
    dict(path="char", alpha=-0.5, beta=0.0, beam=16, T=40, B=1, seed=5, chunk=5),
]


@needs_ref
@pytest.mark.parametrize("cfg", HOOK_CASES, ids=[_case_id(c) for c in HOOK_CASES])
def test_hook_scorer(cfg, monkeypatch):
    """the reference's own Scorer behind the host hook: the kernel does not know alpha, only the terms"""
    which, labels, probs, sl, kw = _inputs(cfg)
    alpha, beta, chunk = kw.pop("alpha"), kw.pop("beta"), kw.pop("chunk", 0)
    if chunk:
        monkeypatch.setenv("CTC_EMU_LM_CHUNK", str(chunk))
    ref = orc.Reference(labels, model_path=PATHS[which], alpha=alpha, beta=beta)
    char = which == "char"
    got = emul.decode_lm(probs, ref.lib, ref.scorer, labels, [] if char else ref.lm_vocabulary(), ref.max_order(),
                         alpha, beta, seq_lens=sl, char_based=char, **kw)
    compare(ref.decode(probs, sl, num_processes=2, **kw), got, None, _case_id(cfg))


SWEEP_PAIRS = [(2.0, 1.0), (-2.0, 1.0), (0.0, 4.0), (-5.0, -4.0)]


@needs_ref
def test_sweep_mixing_signs_word_model():
    """each CTA bounds its keys with its own pair: every slice equals the single-pair decode and the reference"""
    probs = ctc_like_probs(2, 80, 29, seed=5).numpy()
    check_sweep(probs, L29, TEST_ARPA, SWEEP_PAIRS, seq_lens=[80, 1], beam=24)


@needs_ref
def test_sweep_mixing_signs_char_model():
    probs = ctc_like_probs(2, 50, len(LCHAR), seed=35).numpy()
    check_sweep(probs, LCHAR, CHAR_LM, SWEEP_PAIRS, beam=12, cutoff_top_n=10)
