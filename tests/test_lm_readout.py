"""The read-out rescoring of the ARPA scorer (reference DecoderState::decode, ctc_beam_search_decoder.cpp:173-208): the
per-row function the library's read-out kernel runs (ngram_readout_row), compiled for the CPU by
tests/native/emulate_readout.cpp, and the library's host read-out (ctcdec_scorer_rescore_rows with device -1), both
against the reference build's Scorer on adversarial rows.  The float32 score bits must be equal.  CPU only."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from ctcdecode_b200 import _native
from oracle import oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TEST_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
# word-based labels with a multi-byte label, a two-character label and a label with an embedded space
LWORD = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'", "é", "qu", "a b"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu", "x y"]
MODELS = [(TEST_ARPA, LWORD), (TINY, LWORD), (CHAR_LM, LCHAR)]
IDS = ["test.arpa", "tiny_lm", "char_lm"]
PARAMS = [(2.0, 1.0), (1.5, 0.5), (0.7, -1.3), (0.0, 0.0)]

needs_ref = pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)")
_i32p = ctypes.POINTER(ctypes.c_int32)
_SRC = os.path.join(HERE, "native", "emulate_readout.cpp")
_OUT = os.path.join(HERE, "native", "_build", "libctc_emul_readout.so")
_lib = None


def _emu():
    global _lib
    if _lib is None:
        os.makedirs(os.path.dirname(_OUT), exist_ok=True)
        csrc = os.path.join(ROOT, "ctcdecode_b200", "csrc")
        deps = [_SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not (os.path.exists(_OUT) and all(os.path.getmtime(_OUT) >= os.path.getmtime(d) for d in deps)):
            tmp = _OUT + ".%d" % os.getpid()
            subprocess.run(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=off", "-fPIC", "-shared", "-nostdlib++",
                            "-Wno-unused-function", _SRC, "-o", tmp, "-l:libstdc++.so.6", "-lm"], check=True)
            os.replace(tmp, _OUT)
        _lib = ctypes.CDLL(_OUT)
        _lib.emu_readout_rows.restype = ctypes.c_int
        _lib.emu_readout_rows.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_char_p), ctypes.c_int,
                                          ctypes.c_double, ctypes.c_double, _i32p, _i32p, _i32p,
                                          ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return _lib


def _words(path):
    out, section = [], 0
    for line in open(path, encoding="utf-8"):
        line = line.rstrip("\n")
        if line.startswith("\\"):
            section = int(line[1]) if line[1:2].isdigit() else 0
            continue
        if section == 1 and line.strip():
            out.append(line.split()[1])
    return out


def _spell(text, labels):
    """label ids of text, greedily by the single-character labels (characters without one are dropped)"""
    return [labels.index(c) for c in text if c in labels]


def adversarial_rows(path, labels, n_random=300, seed=5):
    """Empty rows; leading, trailing and repeated spaces; words missing from the model; a last word that is only a
    prefix of a dictionary word; the multi-byte, two-character and embedded-space labels; seeded random rows."""
    sp = labels.index(" ")
    words = [w for w in _words(path) if w not in ("<s>", "</s>", "<unk>")]
    specials = [labels.index(x) for x in labels if len(x) > 1 or ord(x[0]) > 127]
    rng = random.Random(seed)
    rows = [[], [sp], [sp, sp, sp], [0], [specials[0]], [specials[-1]], specials]
    for _ in range(40):
        ws = [rng.choice(words) for _ in range(rng.randint(1, 5))]
        text = " ".join(ws)
        rows.append(_spell(text, labels))
        rows.append([sp] + _spell(text, labels))                           # leading space
        rows.append(_spell(text, labels) + [sp] * rng.randint(1, 3))       # trailing spaces
        rows.append(_spell("  ".join(ws), labels))                         # repeated spaces
        w = rng.choice(words)
        rows.append(_spell(text + " " + w[:max(1, len(w) - 1)], labels))   # the last word cut short
        rows.append(_spell(text + " zzqx", labels))                        # a word the model lacks
        ids = _spell(text, labels)
        k = rng.randrange(len(ids) + 1)
        rows.append(ids[:k] + [rng.choice(specials)] + ids[k:])            # é / qu / an embedded space inside
    for _ in range(n_random):
        n = rng.randint(0, 40)
        rows.append([sp if rng.random() < 0.2 else rng.randrange(len(labels)) for _ in range(n)])
    return rows


def pack(rows, K, seed):
    """[B, K, row_stride] tokens, lens, n_results (some utterances hold fewer rows than K) and scores"""
    rng = np.random.default_rng(seed)
    B = (len(rows) + K - 1) // K + 1
    stride = max(1, max(len(r) for r in rows)) + 3
    tok = np.full((B, K, stride), -1, np.int32)
    lens = np.full((B, K), -7, np.int32)
    nres = np.zeros(B, np.int32)
    it = iter(rows)
    for b in range(B):
        for p in range(K if b % 3 else rng.integers(0, K + 1)):
            r = next(it, None)
            if r is None:
                break
            tok[b, p, :len(r)] = r
            lens[b, p] = len(r)
            nres[b] = p + 1
    scores = rng.uniform(0.0, 400.0, (B, K)).astype(np.float32)
    return tok, lens, nres, scores


def reference_readout(ref, labels, tok, lens, nres, scores, alpha, beta):
    """the reference's read-out from its Scorer's two terms, in its own float / double steps (Python floats are IEEE
    doubles without FMA)"""
    f32 = np.float32
    out = scores.copy()
    cb = ref.is_character_based()
    sp = labels.index(" ")
    for b in range(tok.shape[0]):
        for p in range(min(int(nres[b]), tok.shape[1])):
            n = int(lens[b, p])
            ids = (ctypes.c_int32 * max(1, n))(*tok[b, p, :n].tolist())
            arr = ctypes.cast(ids, ctypes.POINTER(ctypes.c_int32))
            ext = f32(-scores[b, p])
            if not cb and n > 0 and int(tok[b, p, n - 1]) != sp:
                s = f32(ref.lib.ref_scorer_cond_from_labels(ref.scorer, arr, n) * alpha)
                s = f32(float(s) + beta)
                ext = f32(ext + s)
            approx = float(ext) - n * beta
            approx -= ref.lib.ref_scorer_sent_from_labels(ref.scorer, arr, n) * alpha
            out[b, p] = f32(-float(f32(approx)))
    return out


def emu_readout(path, labels, alpha, beta, tok, lens, nres, scores):
    out = np.ascontiguousarray(scores.copy())
    lab = (ctypes.c_char_p * len(labels))(*[x.encode() for x in labels])
    B, K, stride = tok.shape
    rc = _emu().emu_readout_rows(path.encode(), lab, len(labels), alpha, beta, tok.ctypes.data_as(_i32p),
                                 lens.ctypes.data_as(_i32p), nres.ctypes.data_as(_i32p),
                                 out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), B, K, stride)
    assert rc == 0
    return out


def lib_readout(handle, tok, lens, nres, scores, device=-1):
    out = np.ascontiguousarray(scores.copy())
    B, K, stride = tok.shape
    _native.check(_native.load().ctcdec_scorer_rescore_rows(handle, tok.ctypes.data, lens.ctypes.data, nres.ctypes.data,
                                                            out.ctypes.data, B, K, stride, device))
    return out


def arpa_scorer(path, labels, alpha, beta):
    lib = _native.load()
    lab = (ctypes.c_char_p * len(labels))(*[s.encode() for s in labels])
    h = ctypes.c_void_p()
    _native.check(lib.ctcdec_scorer_create_arpa(path.encode(), alpha, beta, lab, len(labels), ctypes.byref(h)))
    return h.value


def _same_bits(want, got, rows_of, what):
    bad = np.argwhere(want.view(np.int32) != got.view(np.int32))
    assert bad.size == 0, "%s: %d rows differ, first %s: %r want %r got %r" % (
        what, len(bad), tuple(bad[0]), rows_of(*bad[0]), want[tuple(bad[0])], got[tuple(bad[0])])


@needs_ref
@pytest.mark.parametrize("path,labels", MODELS, ids=IDS)
@pytest.mark.parametrize("alpha,beta", PARAMS)
def test_row_function_and_host_readout_match_reference(path, labels, alpha, beta):
    tok, lens, nres, scores = pack(adversarial_rows(path, labels), 8, seed=int(alpha * 10 + beta * 100) & 0xffff)
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    want = reference_readout(ref, labels, tok, lens, nres, scores, alpha, beta)

    def row(b, p):
        return "".join(labels[i] for i in tok[b, p, :lens[b, p]])
    _same_bits(want, emu_readout(path, labels, alpha, beta, tok, lens, nres, scores), row, "per-row function")
    h = arpa_scorer(path, labels, alpha, beta)
    try:
        _same_bits(want, lib_readout(h, tok, lens, nres, scores), row, "host read-out")
    finally:
        _native.load().ctcdec_scorer_destroy(h)
    skipped = np.arange(tok.shape[1])[None, :] >= nres[:, None]
    assert np.array_equal(want[skipped].view(np.int32), scores[skipped].view(np.int32))


def test_rescore_rows_checks_its_arguments():
    lib = _native.load()
    h = arpa_scorer(TINY, LWORD, 1.0, 0.5)
    try:
        tok = np.zeros((1, 2, 4), np.int32)
        lens = np.array([[2, 5]], np.int32)
        nres = np.array([2], np.int32)
        sc = np.zeros((1, 2), np.float32)
        args = (tok.ctypes.data, lens.ctypes.data, nres.ctypes.data, sc.ctypes.data, 1, 2, 4)
        assert lib.ctcdec_scorer_rescore_rows(h, *args, -1) == -1 and b"length 5" in lib.ctcdec_last_error()
        lens[0, 1] = 1
        tok[0, 1, 0] = len(LWORD)
        assert lib.ctcdec_scorer_rescore_rows(h, *args, -1) == -1 and b"label" in lib.ctcdec_last_error()
        tok[0, 1, 0] = 3
        assert lib.ctcdec_scorer_rescore_rows(h, *args, -1) == 0
        assert lib.ctcdec_scorer_rescore_rows(None, *args, -1) == -1
    finally:
        lib.ctcdec_scorer_destroy(h)


def test_non_blocking_needs_device_outputs_and_the_device_scorer(monkeypatch):
    import ctcdecode_b200
    monkeypatch.delenv("CTCDECODE_B200_SCORER_PROVIDER", raising=False)
    for cls in (ctcdecode_b200.CTCBeamDecoder, ctcdecode_b200.OnlineCTCBeamDecoder):
        with pytest.raises(ValueError, match="device_outputs"):
            cls(LWORD, model_path=TINY, scorer_provider="device", non_blocking=True)
        with pytest.raises(ValueError, match="scorer_provider"):
            cls(LWORD, model_path=TINY, scorer_provider="/nonexistent/provider.so", device_outputs=True,
                non_blocking=True)
        assert cls(LWORD, model_path=TINY, scorer_provider="device", device_outputs=True, non_blocking=True)
        assert cls(LWORD, device_outputs=True, non_blocking=True)  # (no language model: nothing else is needed)
        monkeypatch.setenv("CTCDECODE_B200_SCORER_PROVIDER", "device")
        assert cls(LWORD, model_path=TINY, device_outputs=True, non_blocking=True)
        monkeypatch.delenv("CTCDECODE_B200_SCORER_PROVIDER")
