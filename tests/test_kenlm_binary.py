"""KenLM binary files in the library's own n-gram scorer (ctcdec_scorer_create_arpa, which reads ARPA text and every
binary type KenLM's LoadVirtual reads but REST_PROBING).  The binaries are written when the tests run, by KenLM's own
build_binary (oracle/_ref/build_binary, recipe oracle/build_binary.mk), from the committed ARPA fixtures and from a
seeded synthetic order-6 model.  The authority is the reference's Scorer over KenLM reading the same binary file: hooks,
read-out (the per-row function through tests/native/emulate_readout_file.cpp) and the emulated CTA program
(tests/native/emulate_ngram_file.cpp) must equal it bit for bit.  Then every refusal of a damaged binary is named.
CPU only."""
import ctypes
import itertools
import os
import random
import struct
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from tests import golden_util
from tests.parity import compare
from tests.test_lm_readout import (LCHAR as RLCHAR, LWORD as RLWORD, adversarial_rows, lib_readout, pack,
                                   reference_readout, _same_bits)
from tests.test_ngram_scorer import Arpa, _check, _ngrams, _spell, _spelling_labels, _words

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]
BUILD_BINARY = os.path.join(ROOT, "oracle", "_ref", "build_binary")

# the five binary types the scorer reads: build_binary's arguments before the input file
TYPES = {
    "probing": ["probing"],
    "trie": ["trie"],
    "qtrie": ["-q", "8", "-b", "8", "trie"],
    "atrie": ["-a", "22", "trie"],
    "qatrie": ["-q", "8", "-b", "8", "-a", "22", "trie"],
}
FIXTURES = {"test.arpa": (TEST_ARPA, L29), "tiny_lm": (TINY, L29), "char_lm": (CHAR_LM, LCHAR)}

needs_tools = pytest.mark.skipif(not (orc.reference_available() and os.path.exists(BUILD_BINARY)),
                                 reason="oracle/_ref (reference build and build_binary) not built")


def build_binary(arpa, out_dir, kind, name=None):
    """KenLM's build_binary of `arpa` into out_dir; sorting memory and temporary files stay small and local."""
    out = os.path.join(str(out_dir), "%s.%s" % (name or os.path.basename(arpa), kind))
    if not os.path.exists(out):
        subprocess.run([BUILD_BINARY, "-S", "64M", "-T", str(out_dir)] + TYPES[kind] + [arpa, out], check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return out


def synthetic_arpa(path, seed=2026, order=6, n_words=3000, counts=(40000, 30000, 15000, 8000, 4000)):
    """A seeded order-6 ARPA model of about 100k n-grams over words spelled with L29's letters.  Every n-gram's context
    is in the model; some n-grams whose suffix is a lower n-gram lose that suffix, as SRILM pruning leaves them."""
    rng = random.Random(seed)
    letters = "abcdefghijklmnopqrstuvwxyz'"
    words = set()
    while len(words) < n_words:
        words.add("".join(rng.choice(letters) for _ in range(rng.randint(2, 8))))
    vocab = ["<unk>", "<s>", "</s>"] + sorted(words)
    grams = [[(w,) for w in vocab]]
    for n in range(2, order + 1):
        ctx = [g for g in grams[-1] if g[-1] != "</s>"]
        if n == 2:
            pool = [c + (w,) for c in rng.sample(ctx, len(ctx)) for w in rng.sample(vocab[2:], 20)]
        else:  # c + (w,) whose suffix c[1:] + (w,) is an (n - 1)-gram
            follow = {}
            for g in grams[-1]:
                follow.setdefault(g[:-1], []).append(g[-1])
            pool = [c + (w,) for c in ctx for w in follow.get(c[1:], ())]
        grams.append(sorted(rng.sample(pool, min(len(pool), counts[n - 2]))))
    # SRILM-style pruning: drop some n-grams (2 <= n < order) that are no n-gram's context but the suffix of one
    contexts = set(g[:-1] for level in grams[2:] for g in level)
    for n in range(2, order):
        suffixes = set(g[1:] for g in grams[n])
        pool = sorted(g for g in grams[n - 1] if g in suffixes and g not in contexts)
        drop = set(rng.sample(pool, min(len(pool), 150)))
        grams[n - 1] = [g for g in grams[n - 1] if g not in drop]
    has_ext = set(g[:-1] for level in grams[1:] for g in level)
    with open(path, "w") as f:
        f.write("\\data\\\n")
        for n, level in enumerate(grams, 1):
            f.write("ngram %d=%d\n" % (n, len(level)))
        for n, level in enumerate(grams, 1):
            f.write("\n\\%d-grams:\n" % n)
            for g in level:
                prob = -99.0 if g == ("<s>",) else -round(rng.uniform(0.05, 6.0), 6)
                line = "%g\t%s" % (prob, " ".join(g))
                if n < order and (g in has_ext or rng.random() < 0.3):
                    line += "\t%g" % (0.0 if rng.random() < 0.1 else -round(rng.uniform(0.0, 1.5), 6))
                f.write(line + "\n")
        f.write("\n\\end\\\n")
    return path


@pytest.fixture(scope="module")
def binaries(tmp_path_factory):
    """{(fixture, type): path} for the three fixtures and the synthetic model in all five types"""
    if not (orc.reference_available() and os.path.exists(BUILD_BINARY)):
        pytest.skip("oracle/_ref (reference build and build_binary) not built")
    d = tmp_path_factory.mktemp("kenlm")
    out = {}
    synth = synthetic_arpa(str(d / "synthetic.arpa"))
    for name, path in [(n, p) for n, (p, _) in FIXTURES.items()] + [("synthetic", synth)]:
        out[(name, "arpa")] = path
        for kind in TYPES:
            out[(name, kind)] = build_binary(path, d, kind, name)
    return out


# ---- the CPU emulation harnesses over load_ngram_file (tests/native/emulate_*_file.cpp) ----------------------------

_i32p = ctypes.POINTER(ctypes.c_int32)
_f32p = ctypes.POINTER(ctypes.c_float)
_harness = {}


def _native_lib(name):
    """tests/native/<name>.cpp compiled into tests/native/_build/lib<name>.so (again when a source is newer)"""
    if name not in _harness:
        here = os.path.join(ROOT, "tests", "native")
        src, out = os.path.join(here, name + ".cpp"), os.path.join(here, "_build", "lib%s.so" % name)
        csrc = os.path.join(ROOT, "ctcdecode_b200", "csrc")
        deps = [os.path.join(here, f) for f in os.listdir(here) if f.endswith(".cpp")] + \
            [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps)):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            tmp = out + ".%d" % os.getpid()
            subprocess.run(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=off", "-fPIC", "-shared", "-nostdlib++",
                            "-Wno-unused-function", "-pthread", src, "-o", tmp, "-l:libstdc++.so.6", "-lm"], check=True)
            os.replace(tmp, out)
        _harness[name] = ctypes.CDLL(out)
    return _harness[name]


def emu_decode(probs, labels, path, alpha, beta, seq_lens=None, beam=100, cutoff_prob=1.0, cutoff_top_n=40,
               blank_id=0, log_input=False):
    """the CTA program with the library's own scorer over the model file at path, in the CPU emulation"""
    lib = _native_lib("emulate_ngram_file")
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    B, T, V = probs.shape
    sl = None if seq_lens is None else np.ascontiguousarray(seq_lens, dtype=np.int32)
    tok, ts = np.full((B, beam, T), -1, np.int32), np.full((B, beam, T), -1, np.int32)
    sc, ln = np.zeros((B, beam), np.float32), np.zeros((B, beam), np.int32)
    nres, flags = np.zeros((B,), np.int32), np.zeros((B,), np.int32)
    lab = (ctypes.c_char_p * V)(*[x.encode() for x in labels])
    p = lambda a: a.ctypes.data_as(_i32p)  # noqa: E731
    rc = lib.emu_decode_batch_ngram(
        probs.ctypes.data_as(_f32p), p(sl) if sl is not None else None, B, T, V, beam, ctypes.c_double(cutoff_prob),
        cutoff_top_n, blank_id, int(log_input), 0, 0, path.encode(), ctypes.c_double(alpha), ctypes.c_double(beta),
        lab, p(tok), p(ts), sc.ctypes.data_as(_f32p), p(ln), p(nres), p(flags))
    assert rc == 0, rc
    return dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, n_results=nres, ties=flags)


def emu_readout(path, labels, alpha, beta, tok, lens, nres, scores):
    """the read-out kernel's per-row function, compiled for the CPU, over the model file at path"""
    lib = _native_lib("emulate_readout_file")
    out = np.ascontiguousarray(scores.copy())
    lab = (ctypes.c_char_p * len(labels))(*[x.encode() for x in labels])
    B, K, stride = tok.shape
    rc = lib.emu_readout_rows(path.encode(), lab, len(labels), ctypes.c_double(alpha), ctypes.c_double(beta),
                              tok.ctypes.data_as(_i32p), lens.ctypes.data_as(_i32p), nres.ctypes.data_as(_i32p),
                              out.ctypes.data_as(_f32p), B, K, stride)
    assert rc == 0, rc
    return out


def _close(s):
    s.lib.ctcdec_scorer_destroy(s.handle)
    s.handle = None


# ---- 1. the hooks -------------------------------------------------------------------------------------------------

@needs_tools
@pytest.mark.parametrize("kind", list(TYPES))
@pytest.mark.parametrize("name", list(FIXTURES))
def test_hooks_equal_kenlm_over_the_same_binary(binaries, name, kind):
    """every n-gram of the fixture, spelled as a prefix, cut short and followed by a space; seeded random label rows;
    the accessors"""
    arpa, labels = FIXTURES[name]
    path = binaries[(name, kind)]
    spell_labels = _spelling_labels(arpa)
    mine = Arpa(path, spell_labels)
    assert mine.rc == 0, mine.error
    ref = orc.Reference(spell_labels, model_path=path, alpha=1.0, beta=1.0)
    cb = ref.is_character_based()
    seqs = []
    for ng in _ngrams(arpa):
        ids = _spell(ng, spell_labels, cb)
        seqs += [ids, ids[:-1], ids + [spell_labels.index(" ")]]
    _check(mine, ref, seqs, "%s %s n-grams" % (name, kind))
    _close(mine)

    mine = Arpa(path, labels, 1.5, 0.5)
    assert mine.rc == 0, mine.error
    ref = orc.Reference(labels, model_path=path, alpha=1.5, beta=0.5)
    lib = mine.lib
    assert lib.ctcdec_scorer_max_order(mine.handle) == ref.max_order()
    assert lib.ctcdec_scorer_is_character_based(mine.handle) == ref.is_character_based()
    assert lib.ctcdec_scorer_dict_size(mine.handle) == ref.dict_size()
    words = _words(arpa)
    rng = random.Random(11)
    seqs = [[]]
    for k in range(1500):
        if k % 2:
            seqs.append([rng.randrange(len(labels)) for _ in range(rng.randint(0, 14))])
        else:
            s = " ".join(rng.choice(words) for _ in range(rng.randint(1, 6)))
            s = s[:rng.randint(0, len(s))] if rng.random() < 0.4 else s
            seqs.append([labels.index(c) for c in s if c in labels])
    _check(mine, ref, seqs, "%s %s random rows" % (name, kind))
    _close(mine)


@needs_tools
@pytest.mark.parametrize("kind", list(TYPES))
def test_every_short_sequence_of_test_arpa(binaries, kind):
    """every one-to-three-word sequence over test.arpa's vocabulary: this reaches its n-grams with missing suffixes,
    which build_binary fills in"""
    path = binaries[("test.arpa", kind)]
    labels = _spelling_labels(TEST_ARPA)
    mine = Arpa(path, labels)
    assert mine.rc == 0, mine.error
    ref = orc.Reference(labels, model_path=path, alpha=1.0, beta=1.0)
    vocab = ref.lm_vocabulary()
    assert len(vocab) == 37
    seqs = [_spell(ws, labels, False) for n in (1, 2, 3) for ws in itertools.product(vocab, repeat=n)]
    _check(mine, ref, seqs, "test.arpa %s sequences" % kind)
    _close(mine)


@needs_tools
@pytest.mark.parametrize("name", list(FIXTURES) + ["synthetic"])
def test_probing_binary_equals_its_arpa_source(binaries, name):
    """a probing file holds exactly what the ARPA loader builds: the two scorers agree on every query"""
    arpa = binaries[(name, "arpa")]
    labels = FIXTURES[name][1] if name in FIXTURES else L29
    a, b = Arpa(arpa, labels), Arpa(binaries[(name, "probing")], labels)
    assert a.rc == 0 and b.rc == 0, (a.error, b.error)
    words = [w for w in _words(arpa) if w not in ("<s>", "</s>", "<unk>")]
    cb = a.lib.ctcdec_scorer_is_character_based(a.handle)
    rng = random.Random(3)
    grams = _ngrams(arpa)
    for _ in range(4000):
        ws = list(rng.choice(grams)) if rng.random() < 0.7 else [rng.choice(words) for _ in range(rng.randint(1, 7))]
        ws = [w for w in ws if w not in ("<s>", "</s>")]
        ids = [labels.index(c) for c in (" ".join(ws) if not cb else "".join(ws)) if c in labels]
        for which in ("cond", "sent"):
            assert struct.pack("<d", a.hook(which, ids)) == struct.pack("<d", b.hook(which, ids)), (which, ws)
    _close(a)
    _close(b)


@needs_tools
@pytest.mark.parametrize("kind", list(TYPES))
def test_synthetic_order6_model(binaries, kind):
    """about 20k sampled queries on the order-6 model with pruned suffixes, multi-byte trie fields and probing
    collisions"""
    arpa, path = binaries[("synthetic", "arpa")], binaries[("synthetic", kind)]
    mine = Arpa(path, L29, 1.0, 1.0)
    assert mine.rc == 0, mine.error
    ref = orc.Reference(L29, model_path=path, alpha=1.0, beta=1.0)
    assert mine.lib.ctcdec_scorer_max_order(mine.handle) == ref.max_order() == 6
    assert mine.lib.ctcdec_scorer_dict_size(mine.handle) == ref.dict_size()
    assert mine.lib.ctcdec_scorer_is_character_based(mine.handle) == ref.is_character_based() == 0
    grams = [g for g in _ngrams(arpa) if len(g) >= 2]
    words = [w for w in _words(arpa) if w not in ("<s>", "</s>", "<unk>")]
    rng = random.Random(17)
    seqs = []
    for k in range(10000):
        g = [w for w in rng.choice(grams) if w not in ("<s>", "</s>", "<unk>")]
        if k % 4 == 1:
            g = [rng.choice(words)] + g  # a longer history than the n-gram
        elif k % 4 == 2 and g:
            g[rng.randrange(len(g))] = rng.choice(words)  # one word swapped: a back-off in the middle
        elif k % 4 == 3:
            g = [rng.choice(words) for _ in range(rng.randint(1, 7))]
        ids = _spell(g, L29, False)
        seqs.append(ids if rng.random() < 0.8 else ids + [L29.index(" ")])
    _check(mine, ref, seqs, "synthetic %s" % kind)
    _close(mine)


# ---- 2. the read-out ----------------------------------------------------------------------------------------------

@needs_tools
@pytest.mark.parametrize("kind", ["probing", "qatrie"])
@pytest.mark.parametrize("name", list(FIXTURES))
def test_readout_equals_kenlm(binaries, name, kind):
    """the per-row read-out function (compiled for the CPU) and the library's host read-out on the adversarial rows"""
    path = binaries[(name, kind)]
    labels = RLCHAR if name == "char_lm" else RLWORD
    alpha, beta = 1.5, 0.5
    tok, lens, nres, scores = pack(adversarial_rows(FIXTURES[name][0], labels), 8, seed=23)
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    want = reference_readout(ref, labels, tok, lens, nres, scores, alpha, beta)

    def row(b, p):
        return "".join(labels[i] for i in tok[b, p, :lens[b, p]])
    _same_bits(want, emu_readout(path, labels, alpha, beta, tok, lens, nres, scores), row, "per-row function")
    s = Arpa(path, labels, alpha, beta)
    assert s.rc == 0, s.error
    _same_bits(want, lib_readout(s.handle, tok, lens, nres, scores), row, "host read-out")
    _close(s)


# ---- 3. the emulated CTA program ----------------------------------------------------------------------------------

@needs_tools
@pytest.mark.parametrize("kind", ["probing", "qatrie"])
@pytest.mark.parametrize("name", golden_util.names(lm=True) + golden_util.names_char())
def test_emulated_decode_equals_reference_build(binaries, name, kind):
    """the golden LM inputs decoded by the CTA program in the CPU emulation over a binary, against the reference build
    over the same binary"""
    probs, seq_lens, kw, _gold, alpha, beta = golden_util.load_lm(name)
    char = name.startswith("lmchar_")
    labels, which = (LCHAR, "char_lm") if char else (L29, "tiny_lm")
    path = binaries[(which, kind)]
    want = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta).decode(probs, seq_lens, num_processes=2, **kw)
    got = emu_decode(probs, labels, path, alpha, beta, seq_lens=seq_lens, **kw)
    compare(want, got, None, "%s %s" % (name, kind))


# ---- 4. refusals --------------------------------------------------------------------------------------------------

def _header(data):
    """(order, model type, header bytes) of a binary's bytes"""
    order = data[88]
    mtype = struct.unpack_from("<i", data, 96)[0]
    header = (88 + 20 + 8 * order + 7) // 8 * 8
    return order, mtype, header


def _edit(data, off, fmt, value):
    out = bytearray(data)
    struct.pack_into(fmt, out, off, value)
    return bytes(out)


@needs_tools
def test_refusals_name_the_reason(binaries, tmp_path):
    probing = open(binaries[("test.arpa", "probing")], "rb").read()
    trie = open(binaries[("test.arpa", "trie")], "rb").read()
    order, _, header = _header(probing)
    assert order == 5
    counts = struct.unpack_from("<5Q", probing, 108)
    # test.arpa's probing layout: vocabulary (8 + 12 x buckets), unigrams (counts[0] + 1) x 8, then the tables
    mult = struct.unpack_from("<f", probing, 92)[0]
    buckets = [max(c + 1, int(np.float32(mult) * np.float32(c))) for c in counts]
    bigrams_at = header + 8 + 12 * buckets[0] + (counts[0] + 1) * 8
    overfull = bytearray(probing)
    for b in range(buckets[1]):
        if struct.unpack_from("<Q", overfull, bigrams_at + 16 * b)[0] == 0:
            struct.pack_into("<Q", overfull, bigrams_at + 16 * b, 0x1234567 + b)
    trie_counts = struct.unpack_from("<5Q", trie, 108)  # (with the entries build_binary added for pruned suffixes)
    uni_at = header + 8 + 8 * trie_counts[0]  # the trie's unigrams: (prob, backoff, next) after the sorted vocabulary
    cases = [
        ("truncated", probing[:60], "truncated"),
        ("truncated_tables", probing[:header + 40], "truncated"),
        ("incomplete", b"mmap lm http://kheafield.com/code incomplete\n" + probing[46:], "did not finish building"),
        ("version", probing.replace(b"format version 5", b"format version 4", 1), "format version 4"),
        ("sanity_float", _edit(probing, 60, "<f", 2.0), "test values"),
        ("rest_probing", _edit(probing, 96, "<i", 1), "REST_PROBING"),
        ("model_type", _edit(probing, 96, "<i", 9), "unknown model type 9"),
        ("search_version", _edit(trie, 104, "<I", 7), "search version 7"),
        ("order7", _edit(probing, 88, "<B", 7), "order 7 is above 6"),
        ("order1", _edit(probing, 88, "<B", 1), "order 1"),
        ("no_vocabulary", _edit(probing, 100, "<B", 0), "no vocabulary strings"),
        ("vocabulary_count", _edit(probing, header + 4, "<I", counts[0] + 5), "the vocabulary has"),
        ("strings_cut", probing[:-8], "vocabulary string"),
        ("overfull_probing", bytes(overfull), "no empty bucket"),
        ("trie_pointer", _edit(trie, uni_at + 16 * 3 + 8, "<Q", 1 << 40), "trie pointer"),
        ("trie_pointer_past", _edit(trie, uni_at + 16 * trie_counts[0] + 8, "<Q", trie_counts[1] + 3), "points past"),
    ]
    for name, data, reason in cases:
        p = tmp_path / (name + ".binary")
        p.write_bytes(data)
        s = Arpa(str(p), L29)
        assert s.rc == -2, (name, s.rc, s.error)
        assert "KenLM binary" in s.error and reason in s.error, (name, s.error)
        assert s.handle is None
        good = Arpa(binaries[("test.arpa", "qatrie")], L29)  # and the next model loads
        assert good.rc == 0, good.error
        _close(good)


@needs_tools
@pytest.mark.parametrize("kind", ["probing", "trie"])
def test_missing_sentence_markers_are_refused(binaries, tmp_path, kind):
    data = open(binaries[("test.arpa", kind)], "rb").read()
    for marker, other in ((b"\0</s>\0", b"\0</x>\0"), (b"\0<s>\0", b"\0<x>\0")):
        p = tmp_path / "no_marker.binary"
        p.write_bytes(data.replace(marker, other))
        s = Arpa(str(p), L29)
        assert s.rc == -2 and "no %s" % marker.strip(b"\0").decode() in s.error, (kind, s.error)
