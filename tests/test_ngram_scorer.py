"""The library's own ARPA scorer (ctcdec_scorer_create_arpa): its hooks against the reference Scorer over KenLM, bit for
bit, and the refusals of models it cannot reproduce exactly.  CPU only: the hooks are host code."""
import ctypes
import itertools
import os
import random
import struct

import pytest

from ctcdecode_b200 import _native
from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]

needs_ref = pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)")


def _words(path):
    """The unigrams of an ARPA file, in file order."""
    out, section = [], 0
    for line in open(path, encoding="utf-8"):
        line = line.rstrip("\n")
        if line.startswith("\\"):
            section = int(line[1]) if line[1:2].isdigit() else 0
            continue
        if section == 1 and line.strip():
            out.append(line.split()[1])
    return out


def _ngrams(path):
    out, section = [], 0
    for line in open(path, encoding="utf-8"):
        line = line.rstrip("\n")
        if line.startswith("\\"):
            section = int(line[1]) if line[1:2].isdigit() else 0
            continue
        if section and line.strip():
            out.append(line.split()[1:1 + section])
    return out


def _spelling_labels(path):
    """Blank, every character of the model's words, and the space: labels that spell every word of the model."""
    chars = sorted({c for w in _words(path) for c in w})
    return ["_"] + chars + [" "]


class Arpa(object):
    def __init__(self, path, labels, alpha=1.0, beta=1.0):
        self.lib = _native.load()
        self.labels = list(labels)
        lab = (ctypes.c_char_p * len(labels))(*[s.encode() for s in labels])
        h = ctypes.c_void_p()
        self.rc = self.lib.ctcdec_scorer_create_arpa(path.encode(), alpha, beta, lab, len(labels), ctypes.byref(h))
        self.error = self.lib.ctcdec_last_error().decode() if self.rc else ""
        self.handle = h.value

    def hook(self, which, ids):
        arr = (ctypes.c_int32 * max(1, len(ids)))(*ids)
        out = ctypes.c_double()
        fn = self.lib.ctcdec_scorer_cond_log_prob if which == "cond" else self.lib.ctcdec_scorer_sent_log_prob
        _native.check(fn(self.handle, arr, len(ids), ctypes.byref(out)))
        return out.value

    def __del__(self):
        if getattr(self, "handle", None):
            self.lib.ctcdec_scorer_destroy(self.handle)


def _ref_hook(ref, which, ids):
    arr = (ctypes.c_int32 * max(1, len(ids)))(*ids)
    fn = ref.lib.ref_scorer_cond_from_labels if which == "cond" else ref.lib.ref_scorer_sent_from_labels
    return fn(ref.scorer, ctypes.cast(arr, ctypes.POINTER(ctypes.c_int32)), len(ids))


def _bits(x):
    return struct.pack("<d", x)


def _check(mine, ref, seqs, what):
    bad = []
    for ids in seqs:
        for which in ("cond", "sent"):
            a, b = mine.hook(which, ids), _ref_hook(ref, which, ids)
            if _bits(a) != _bits(b):
                bad.append((which, "".join(mine.labels[i] for i in ids), a, b))
    assert not bad, "%s: %d mismatches, first %s" % (what, len(bad), bad[:5])


def _spell(words, labels, character_based):
    sep = [] if character_based else [labels.index(" ")]
    ids = []
    for k, w in enumerate(words):
        if k and sep:
            ids += sep
        ids += [labels.index(c) for c in w]
    return ids


FIXTURES = [(TEST_ARPA, L29), (TINY, L29), (CHAR_LM, LCHAR)]


@needs_ref
@pytest.mark.parametrize("path,labels", FIXTURES, ids=["test.arpa", "tiny_lm", "char_lm"])
def test_accessors_match_reference(path, labels):
    mine = Arpa(path, labels, 1.5, 0.5)
    assert mine.rc == 0, mine.error
    ref = orc.Reference(labels, model_path=path, alpha=1.5, beta=0.5)
    lib = mine.lib
    assert lib.ctcdec_scorer_max_order(mine.handle) == ref.max_order()
    assert lib.ctcdec_scorer_is_character_based(mine.handle) == ref.is_character_based()
    assert lib.ctcdec_scorer_dict_size(mine.handle) == ref.dict_size()
    assert lib.ctcdec_scorer_reset_params(mine.handle, 0.25, 2.0) == 0


@needs_ref
@pytest.mark.parametrize("path", [TEST_ARPA, TINY, CHAR_LM], ids=["test.arpa", "tiny_lm", "char_lm"])
def test_every_ngram_of_the_model(path):
    """every n-gram of the file, spelled with labels that can spell all its words, as a prefix (and the prefix with its
    last word cut short, and followed by a space)"""
    labels = _spelling_labels(path)
    mine = Arpa(path, labels)
    assert mine.rc == 0, mine.error
    ref = orc.Reference(labels, model_path=path, alpha=1.0, beta=1.0)
    cb = ref.is_character_based()
    seqs = []
    for ng in _ngrams(path):
        ids = _spell(ng, labels, cb)
        seqs += [ids, ids[:-1], ids + [labels.index(" ")]]
    _check(mine, ref, seqs, os.path.basename(path))


@needs_ref
def test_every_history_word_pair_of_test_arpa():
    """every (history, word) pair over test.arpa's vocabulary with histories up to 2 words (each word also as the
    "<s>" padding the reference writes), and a seeded sample with histories up to the model's order"""
    labels = _spelling_labels(TEST_ARPA)
    mine = Arpa(TEST_ARPA, labels)
    ref = orc.Reference(labels, model_path=TEST_ARPA, alpha=1.0, beta=1.0)
    vocab = ref.lm_vocabulary()
    assert len(vocab) == 37
    seqs = []
    for n in (1, 2, 3):
        for ws in itertools.product(vocab, repeat=n):
            seqs.append(_spell(ws, labels, False))
    rng = random.Random(7)
    for _ in range(3000):
        ws = [rng.choice(vocab) for _ in range(rng.randint(4, 6))]
        seqs.append(_spell(ws, labels, False))
    _check(mine, ref, seqs, "test.arpa pairs")


@needs_ref
@pytest.mark.parametrize("path,labels", FIXTURES, ids=["test.arpa", "tiny_lm", "char_lm"])
def test_random_label_sequences(path, labels):
    """seeded random prefixes over the decoder's labels: OOV words, partial words, empty prefixes, runs of spaces"""
    mine = Arpa(path, labels)
    ref = orc.Reference(labels, model_path=path, alpha=1.0, beta=1.0)
    words = [w for w in _words(path)]
    rng = random.Random(11)
    seqs = [[]]
    for k in range(3000):
        if k % 2:
            seqs.append([rng.randrange(len(labels)) for _ in range(rng.randint(0, 14))])
        else:
            s = " ".join(rng.choice(words) for _ in range(rng.randint(1, 6)))
            s = s[:rng.randint(0, len(s))] if rng.random() < 0.4 else s
            seqs.append([labels.index(c) for c in s if c in labels])
    _check(mine, ref, seqs, os.path.basename(path))


# ---- refusals ----------------------------------------------------------------------------------------------------

GOOD = """\\data\\
ngram 1=5
ngram 2=3
ngram 3=1

\\1-grams:
-1.0\t<unk>\t0
-99\t<s>\t-0.5
-1.2\t</s>
-0.7\tab\t-0.3
-0.9\tba\t-0.2

\\2-grams:
-0.4\t<s> ab\t-0.1
-0.5\tab ba
-0.6\tba </s>

\\3-grams:
-0.2\t<s> ab ba

\\end\\
"""

L_AB = ["_", "a", "b", " "]


def _write(tmp_path, name, text, mode="w"):
    p = tmp_path / name
    if mode == "wb":
        p.write_bytes(text)
    else:
        p.write_text(text)
    return str(p)


def test_crafted_good_model_is_accepted(tmp_path):
    s = Arpa(_write(tmp_path, "good.arpa", GOOD), L_AB)
    assert s.rc == 0, s.error
    assert s.lib.ctcdec_scorer_max_order(s.handle) == 3
    assert s.lib.ctcdec_scorer_dict_size(s.handle) == 2


@pytest.mark.parametrize("name,text,reason", [
    ("binary", b"mmap lm http://kheafield.com/code\0\0\0\1\2\3", "KenLM binary"),
    ("not_arpa", "hello world\n", "not an ARPA text file"),
    ("order7", "\\data\\\n" + "".join("ngram %d=1\n" % n for n in range(1, 8)) + "\n", "order 7 is above 6"),
    ("too_few", GOOD.replace("ngram 2=3", "ngram 2=4"), "counts disagree"),
    ("too_many", GOOD.replace("ngram 3=1", "ngram 3=0"), "counts disagree"),
    ("missing_context", GOOD.replace("-0.2\t<s> ab ba", "-0.2\tba ab ba"), "context"),
    ("positive", GOOD.replace("-0.5\tab ba", "0.5\tab ba"), "positive log-prob"),
    ("nan_prob", GOOD.replace("-0.5\tab ba", "nan\tab ba"), "non-finite log-prob"),
    ("inf_backoff", GOOD.replace("-0.7\tab\t-0.3", "-0.7\tab\t-inf"), "non-finite backoff"),
    ("no_bos", GOOD.replace("ngram 1=5", "ngram 1=4").replace("-99\t<s>\t-0.5\n", "")
                   .replace("ngram 2=3", "ngram 2=2").replace("-0.4\t<s> ab\t-0.1\n", "")
                   .replace("ngram 3=1", "ngram 3=0").replace("-0.2\t<s> ab ba\n", ""), "no <s>"),
    ("unknown_word", GOOD.replace("-0.5\tab ba", "-0.5\tab cd"), "is not a unigram"),
])
def test_refusals_name_the_reason(tmp_path, name, text, reason):
    s = Arpa(_write(tmp_path, name + ".arpa", text, "wb" if isinstance(text, bytes) else "w"), L_AB)
    assert s.rc == -2, (s.rc, s.error)   # CTCDEC_E_UNSUPPORTED
    assert reason in s.error, s.error
    assert s.handle is None
    good = Arpa(_write(tmp_path, "after.arpa", GOOD), L_AB)   # and the next model loads
    assert good.rc == 0, good.error


def test_missing_file_is_invalid(tmp_path):
    s = Arpa(str(tmp_path / "nope.arpa"), L_AB)
    assert s.rc == -1 and "cannot open" in s.error


def test_diagnostic_hooks_check_labels():
    s = Arpa(TINY, L29)
    out = ctypes.c_double()
    arr = (ctypes.c_int32 * 2)(1, 29)
    assert s.lib.ctcdec_scorer_cond_log_prob(s.handle, arr, 2, ctypes.byref(out)) == -1
    assert s.lib.ctcdec_scorer_sent_log_prob(None, arr, 1, ctypes.byref(out)) == -1


def test_workspace_holds_the_lm_histories():
    """ctcdec_lm_workspace_bytes adds B x (1 + beam x T) x (order - 1) x 4 bytes of per-node LM histories (config 5 at
    order 5: about 102 MB) and refuses them beyond 64 GiB"""
    s = Arpa(TEST_ARPA, L29)
    lib = s.lib
    cfg = _native.Config(29, 100, 0, 0, 40, 1.0)
    n, m = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), s.handle, 64, 1000, ctypes.byref(n)) == 0
    assert lib.ctcdec_workspace_bytes(ctypes.byref(cfg), 64, 1000, ctypes.byref(m)) == 0
    hist = 64 * (1 + 100 * 1000) * 4 * 4
    assert n.value - m.value >= hist + 2 * 64 * (1 + 100 * 1000) * 4, (n.value, m.value)
    assert lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), s.handle, 264, 170000, ctypes.byref(n)) == -2
    assert b"LM histories" in lib.ctcdec_last_error()
