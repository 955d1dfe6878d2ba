"""KenLM trie files searched where they are (layout kNgramKenlmTrie): the loader keeps a trie file's search region
byte for byte and the one __host__ __device__ walk (ngram_lm.h ngram_trie_step) searches it, in the host hooks, the
read-out function and the emulated CTA program alike.  The authority is the reference's Scorer over KenLM reading the
same file.  The fixture is a seeded *wide* order-5 model: more than 2^16 words (17-bit word ids), nodes with thousands
of children next to single-child and childless ones, Bhiksha-compressed pointers in its array tries.  Also the
diagnostic ctcdec_scorer_table_bytes, and the refusals of the trie validation pass.  CPU only."""
import ctypes
import os
import random
import struct

import numpy as np
import pytest

from ctcdecode_b200 import _native
from ctcdecode_b200.scorer import ArpaScorer
from ctcdecode_b200.synth import text_probs
from oracle import oracle as orc
from tests.parity import compare
from tests.test_kenlm_binary import (FIXTURES, L29, TYPES, Arpa, _check, _close, _header, _ngrams, _words, binaries,  # noqa: F401
                                     build_binary, emu_decode, emu_readout, needs_tools)
from tests.test_lm_readout import pack, reference_readout, _same_bits

TRIES = ["trie", "qtrie", "atrie", "qatrie"]
LETTERS = "abcdefghijklmnopqrstuvwxyz'"


def wide_arpa(path, seed=5, n_words=70000, hubs=6, hub_preds=2500, bigrams=120000,
              counts=(160000, 120000, 60000)):
    """A seeded order-5 ARPA model over n_words words spelled with L29's letters.  A few hub words follow thousands of
    words, so their nodes in the reversed trie have thousands of children; most words have none or one.  Every
    n-gram's context and suffix are in the model."""
    rng = random.Random(seed)
    words = set()
    while len(words) < n_words:
        words.add("".join(rng.choice(LETTERS) for _ in range(rng.randint(3, 8))))
    vocab = ["<unk>", "<s>", "</s>"] + sorted(words)
    real = vocab[3:]
    big = set()
    for h in rng.sample(real, hubs):
        big.update((w, h) for w in rng.sample(real, hub_preds))
    while len(big) < bigrams + hubs * hub_preds:
        big.add((rng.choice(real), rng.choice(real)))
    big.update(("<s>", w) for w in rng.sample(real, 2000))
    big.update((w, "</s>") for w in rng.sample(real, 2000))
    grams = [[(w,) for w in vocab], sorted(big)]
    for n in range(3, 6):  # c + (w,): context c and suffix c[1:] + (w,) both (n - 1)-grams
        follow = {}
        for g in grams[-1]:
            follow.setdefault(g[:-1], []).append(g[-1])
        pool = [c + (w,) for c in grams[-1] if c[-1] != "</s>" for w in follow.get(c[1:], ())]
        grams.append(sorted(rng.sample(pool, min(len(pool), counts[n - 3]))))
    has_ext = set(g[:-1] for level in grams[1:] for g in level)
    with open(path, "w") as f:
        f.write("\\data\\\n")
        for n, level in enumerate(grams, 1):
            f.write("ngram %d=%d\n" % (n, len(level)))
        for n, level in enumerate(grams, 1):
            f.write("\n\\%d-grams:\n" % n)
            for g in level:
                prob = -99.0 if g == ("<s>",) else -round(rng.uniform(0.05, 7.0), 6)
                line = "%g\t%s" % (prob, " ".join(g))
                if n < 5 and (g in has_ext or rng.random() < 0.3):
                    line += "\t%g" % (0.0 if rng.random() < 0.1 else -round(rng.uniform(0.0, 1.5), 6))
                f.write(line + "\n")
        f.write("\n\\end\\\n")
    return path, grams


@pytest.fixture(scope="module")
def wide(tmp_path_factory):
    """(ARPA path, n-grams by order, {type: path}) of the wide model in the four trie types and as a probing file"""
    if not (orc.reference_available() and os.path.exists(os.path.join(os.path.dirname(orc.__file__), "_ref",
                                                                       "build_binary"))):
        pytest.skip("oracle/_ref (reference build and build_binary) not built")
    d = tmp_path_factory.mktemp("wide")
    arpa, grams = wide_arpa(str(d / "wide.arpa"))
    return arpa, grams, {kind: build_binary(arpa, d, kind, "wide") for kind in TRIES + ["probing"]}


# ---- the file layout, recomputed from the header (KenLM lm/trie.cc, lm/bhiksha.cc) -----------------------------------

def _required_bits(v):
    return v.bit_length()


def _chop(max_offset, max_next, configured=22):
    required = _required_bits(max_next)
    best, lowest = 0, None
    for chop in range(min(required, configured) + 1):
        change = (max_next >> (required - chop)) * 64 - max_offset * chop
        if lowest is None or change < lowest:
            lowest, best = change, chop
    return best


def _layout(data):
    """counts, the unigram array's offset, and per middle order (2..N-1) its entry width, chop, offset-array offset and
    length, and entry 0's byte offset"""
    order, mtype, header = _header(data)
    counts = struct.unpack_from("<%dQ" % order, data, 108)
    quant, array = mtype in (3, 5), mtype in (4, 5)
    at = header + 8 + 8 * counts[0]
    if quant:
        pb, bb = data[at + 1], data[at + 2]
        at += (order - 2) * (((1 << bb) + (1 << pb)) * 4) + (1 << pb) * 4 + 8
    uni_at = at
    at += (counts[0] + 2) * 16
    bh_bits = data[at + 1] if array and order > 2 else 0
    middles = {}
    for n in range(2, order):
        entries, max_next = counts[n - 1], counts[n]
        inline, bhiksha, chop, n_off = _required_bits(max_next), 0, 0, 0
        if array:
            chop = _chop(entries + 1, max_next, bh_bits)
            n_off = (max_next >> (_required_bits(max_next) - chop)) + 1
            bhiksha = 8 * (1 + n_off) + 7
            inline = _required_bits(max_next) - chop
        total = _required_bits(counts[0]) + ((pb + bb) if quant else 63) + inline
        middles[n] = dict(total=total, chop=chop, offsets=(at + 7) // 8 * 8 + 8, n_offsets=n_off, base=at + bhiksha,
                          word_bits=_required_bits(counts[0]))
        at += bhiksha + ((1 + entries) * total + 7) // 8 + 8
    return counts, uni_at, middles


def _get_bits(data, bit, width):
    v = int.from_bytes(data[bit // 8: bit // 8 + 16], "little") >> (bit % 8)
    return v & ((1 << width) - 1)


def _set_bits(data, bit, width, value):
    out = bytearray(data)
    lo = bit // 8
    v = int.from_bytes(out[lo: lo + 16], "little")
    mask = ((1 << width) - 1) << (bit % 8)
    v = (v & ~mask) | ((value << (bit % 8)) & mask)
    out[lo: lo + 16] = v.to_bytes(16, "little")
    return bytes(out)


@needs_tools
def test_wide_model_exercises_the_layout(wide):
    """the fixture is what it claims: 17-bit word ids, unquantized middle entries wider than 64 bits, array tries that
    move pointer bits to the offset array, and nodes with thousands of children, one child and none"""
    arpa, grams, paths = wide
    counts, _, middles = _layout(open(paths["trie"], "rb").read())
    assert counts[0] > 1 << 16 and middles[2]["word_bits"] >= 17
    assert 2e5 <= sum(counts) <= 1e6, counts
    assert all(m["total"] > 64 for m in middles.values()), middles
    for kind in ("atrie", "qatrie"):
        _, _, am = _layout(open(paths[kind], "rb").read())
        assert all(m["chop"] > 0 for m in am.values()), (kind, am)
    for n in (2, 3, 4):  # children of a reversed-trie node: the n-grams ending in it, one older word each
        kids = {}
        for g in grams[n - 1]:
            kids[g[1:]] = kids.get(g[1:], 0) + 1
        sizes = sorted(kids.values())
        assert sizes[0] == 1 and sizes[-1] >= 100, (n, sizes[-5:])
        assert len(kids) < len(grams[n - 2]), n  # parents without children: empty ranges


def _queries(grams, words, rng, count=2500):
    """word sequences that end in a stored n-gram of every order, in one with its oldest word swapped (a miss at that
    order), in a longer history, and with OOV words"""
    seqs = []
    for k in range(count):
        n = 1 + k % 5
        g = list(rng.choice(grams[n - 1]))
        mode = (k // 5) % 4
        if mode == 1 and n > 1:
            g[0] = rng.choice(words)
        elif mode == 2:
            g = [rng.choice(words) for _ in range(rng.randint(1, 3))] + g
        elif mode == 3:
            g[rng.randrange(len(g))] = "".join(rng.choice(LETTERS) for _ in range(10))  # (10 letters: never a word)
        seqs.append([w for w in g if w not in ("<s>", "</s>", "<unk>")])
    return seqs


def _spell_words(ws):
    return [L29.index(c) for c in " ".join(ws)]


@needs_tools
@pytest.mark.parametrize("kind", TRIES)
def test_wide_hooks_equal_kenlm(wide, kind):
    arpa, grams, paths = wide
    words = [w for w in _words(arpa) if w not in ("<s>", "</s>", "<unk>")]
    mine = Arpa(paths[kind], L29, 1.0, 1.0)
    assert mine.rc == 0, mine.error
    ref = orc.Reference(L29, model_path=paths[kind], alpha=1.0, beta=1.0)
    assert mine.lib.ctcdec_scorer_max_order(mine.handle) == ref.max_order() == 5
    rng = random.Random(TRIES.index(kind))
    seqs = []
    for ws in _queries(grams, words, rng):
        ids = _spell_words(ws)
        seqs += [ids, ids + [L29.index(" ")]]
    _check(mine, ref, seqs, "wide %s" % kind)
    _close(mine)


@needs_tools
@pytest.mark.parametrize("kind", TRIES)
def test_wide_readout_and_emulated_decode_equal_reference(wide, kind):
    """the read-out rows (per-row function compiled for the CPU) and the emulated CTA program over the wide model's
    file, against the reference build over the same file"""
    arpa, grams, paths = wide
    path = paths[kind]
    words = [w for w in _words(arpa) if w not in ("<s>", "</s>", "<unk>")]
    rng = random.Random(7)
    rows = []
    for ws in _queries(grams, words, rng, 200):
        s = " ".join(ws)
        rows.append(_spell_words([s if rng.random() < 0.7 else s[:rng.randint(0, len(s))]]))
    tok, lens, nres, scores = pack(rows, 8, seed=29)
    ref = orc.Reference(L29, model_path=path, alpha=1.5, beta=0.5)
    want = reference_readout(ref, L29, tok, lens, nres, scores, 1.5, 0.5)

    def row(b, p):
        return "".join(L29[i] for i in tok[b, p, :lens[b, p]])
    _same_bits(want, emu_readout(path, L29, 1.5, 0.5, tok, lens, nres, scores), row, "wide %s read-out" % kind)

    texts = [" ".join(rng.choice(grams[4])) for _ in range(3)]
    probs = text_probs(texts, L29, 160, seed=31).numpy()
    kw = dict(beam=24, cutoff_prob=1.0, cutoff_top_n=40)
    want = orc.Reference(L29, model_path=path, alpha=1.2, beta=0.4).decode(probs, None, num_processes=2, **kw)
    got = emu_decode(probs, L29, path, 1.2, 0.4, **kw)
    compare(want, got, None, "wide %s emulated decode" % kind)


@needs_tools
def test_table_bytes(binaries, wide):
    """a trie file's n-gram data on the device is at most the file; a probing file's is its own tables, ARPA text's the
    full-key tables"""
    arpa, _, paths = wide
    files = [(n, k, binaries[(n, k)]) for n in list(FIXTURES) + ["synthetic"] for k in TYPES]
    files += [("wide", k, paths[k]) for k in TRIES + ["probing"]]
    for name, kind, path in files:
        data = open(path, "rb").read()
        order, _, header = _header(data)
        counts = struct.unpack_from("<%dQ" % order, data, 108)
        labels = FIXTURES[name][1] if name in FIXTURES else L29
        s = ArpaScorer(labels, path, 1.0, 1.0)
        got = s.table_bytes()
        if kind == "probing":
            mult = struct.unpack_from("<f", data, 92)[0]
            words = struct.unpack_from("<I", data, header + 4)[0]
            want = 8 * words
            for n in range(2, order + 1):
                buckets = max(counts[n - 1] + 1, int(np.float32(mult) * np.float32(counts[n - 1])))
                want += (buckets * (16 if n < order else 12) + 7) // 8 * 8
            assert got == want, (name, kind, got, want)
        else:
            assert got <= len(data), (name, kind, got, len(data))
            if name == "wide":  # several times smaller than the full-key tables of the same n-grams
                assert got * 4 < 32 * 2 * sum(counts[1:]), (kind, got)
        s.release()
    for name, path in [(n, p) for n, (p, _) in FIXTURES.items()] + [("synthetic", binaries[("synthetic", "arpa")])]:
        # ARPA text: unigrams, then the tables of the n-grams the file lists plus the suffixes KenLM fills in; the
        # probing file of the same model counts those (its header's counts)
        data = open(binaries[(name, "probing")], "rb").read()
        order, _, header = _header(data)
        counts = struct.unpack_from("<%dQ" % order, data, 108)
        words = struct.unpack_from("<I", data, header + 4)[0]
        want = 8 * words
        for c in counts[1:]:
            cap = 2
            while cap < 2 * c:
                cap *= 2
            want += 32 * cap
        labels = FIXTURES[name][1] if name in FIXTURES else L29
        s = ArpaScorer(labels, path, 1.0, 1.0)
        assert s.table_bytes() == want, (name, s.table_bytes(), want)
        s.release()


def test_table_bytes_of_a_hook_scorer_is_unsupported():
    lib = _native.load()
    cond = ctypes.CFUNCTYPE(ctypes.c_double, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.c_int)(
        lambda c, l, n: -1.0)
    hooks = _native.ScorerHooks(None, ctypes.cast(cond, ctypes.c_void_p).value, ctypes.cast(cond, ctypes.c_void_p).value)
    lab = (ctypes.c_char_p * 3)(b"_", b"a", b"b")
    h = ctypes.c_void_p()
    assert lib.ctcdec_scorer_create(ctypes.byref(hooks), 1.0, 0.5, lab, 3, None, 0, 3, 1, ctypes.byref(h)) == 0
    n = ctypes.c_size_t(7)
    assert lib.ctcdec_scorer_table_bytes(h, ctypes.byref(n)) == -2 and n.value == 7
    assert lib.ctcdec_scorer_table_bytes(None, ctypes.byref(n)) == -1
    assert lib.ctcdec_scorer_destroy(h) == 0


# ---- refusals of the validation pass --------------------------------------------------------------------------------

def _node_with_children(data, counts, uni_at, at_least):
    """(first child, end) of the first bigram node (a unigram's children) with at least `at_least` children"""
    for w in range(counts[0]):
        a = struct.unpack_from("<Q", data, uni_at + 16 * w + 8)[0]
        b = struct.unpack_from("<Q", data, uni_at + 16 * (w + 1) + 8)[0]
        if b - a >= at_least:
            return a, b
    raise AssertionError("no node with %d children" % at_least)


@needs_tools
def test_trie_validation_refusals(wide, tmp_path):
    """a word id past the vocabulary, two words out of order in one node, a Bhiksha offset that decreases: each is
    refused with its reason, and a good file loads after each"""
    _, _, paths = wide
    trie = open(paths["trie"], "rb").read()
    counts, uni_at, middles = _layout(trie)
    m = middles[2]
    a, b = _node_with_children(trie, counts, uni_at, 3)
    wb, total = m["word_bits"], m["total"]
    first = _get_bits(trie, 8 * m["base"] + a * total, wb)
    second = _get_bits(trie, 8 * m["base"] + (a + 1) * total, wb)
    assert first < second
    atrie = open(paths["atrie"], "rb").read()
    _, _, am = _layout(atrie)
    off, n_off = am[2]["offsets"], am[2]["n_offsets"]
    assert n_off >= 3
    offsets = struct.unpack_from("<%dQ" % n_off, atrie, off)
    assert offsets[0] == 0 and list(offsets) == sorted(offsets)
    j = next(j for j in range(1, n_off) if offsets[j] > 0)
    cases = [
        ("word_past_vocabulary", _set_bits(trie, 8 * m["base"] + (b - 1) * total, wb, (1 << wb) - 1),
         "a trie word id of order 2 is outside the vocabulary"),
        ("words_out_of_order", _set_bits(trie, 8 * m["base"] + (a + 1) * total, wb, first),
         "trie words of order 2 out of order"),
        ("offset_decreases", atrie[:off + 8 * j] + struct.pack("<Q", offsets[j] - 1 if j + 1 == n_off else
                                                               offsets[j + 1] + 1) + atrie[off + 8 * j + 8:],
         "array-compressed pointers out of order"),
    ]
    assert (1 << wb) - 1 >= counts[0] + 1
    for name, data, reason in cases:
        p = tmp_path / (name + ".binary")
        p.write_bytes(data)
        s = Arpa(str(p), L29)
        assert s.rc == -2, (name, s.rc, s.error)
        assert "KenLM binary" in s.error and reason in s.error, (name, s.error)
        assert s.handle is None
        good = Arpa(paths["qatrie"], L29)
        assert good.rc == 0, good.error
        _close(good)
