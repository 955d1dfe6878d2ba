"""KenLM binary files in the device n-gram scorer on the H100 (-m gpu).  The binaries are written when the tests run by
KenLM's build_binary (tests/test_kenlm_binary.py); a probing file's tables are searched in HBM as they are, a trie is
unpacked on load.  Every decode over a binary must equal, bit for bit, the hook scorer over the same binary (the
provider library: the reference's Scorer over KenLM) and the reference build over it."""
import os
import random

import numpy as np
import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200 import _native
from ctcdecode_b200.synth import ctc_like_probs, text_probs
from oracle import oracle as orc
from tests import golden_util
from tests.parity import compare
from tests.test_gpu_lm_async import _async, _blocking, _stream_decode
from tests.test_gpu_ngram_scorer import _dec, _hook, _logits, _res, _same
from tests.test_kenlm_binary import BUILD_BINARY, L29, LCHAR, TYPES, _words, binaries  # noqa: F401 (a fixture)
from tests.test_lm import c5_text_probs

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)"),
    pytest.mark.skipif(not os.path.exists(orc.PROVIDER), reason="scorer provider (make -C oracle provider) not built"),
    pytest.mark.skipif(not os.path.exists(BUILD_BINARY),
                       reason="build_binary (make -C oracle -f build_binary.mk build_binary) not built"),
]

TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran"]
TWO = ["probing", "qatrie"]


@pytest.mark.parametrize("kind", list(TYPES))
@pytest.mark.parametrize("name", golden_util.names(lm=True) + golden_util.names_char())
def test_fixtures_through_every_entry(binaries, name, kind):
    """the golden LM inputs through the host, device and asynchronous entries over a binary, against the hook scorer
    and the reference build over the same binary"""
    probs, seq_lens, kw, _gold, alpha, beta = golden_util.load_lm(name)
    labels, which = (LCHAR, "char_lm") if name.startswith("lmchar_") else (L29, "tiny_lm")
    model = binaries[(which, kind)]
    opts = dict(cutoff_top_n=kw["cutoff_top_n"], cutoff_prob=kw["cutoff_prob"], log_probs_input=kw["log_input"])
    sl = None if seq_lens is None else torch.as_tensor(seq_lens)
    dec = _dec(labels, model, alpha, beta, kw["beam"], **opts)
    host = _res(dec, dec.decode(torch.from_numpy(probs), sl))
    ref = orc.Reference(labels, model_path=model, alpha=alpha, beta=beta)
    compare(ref.decode(probs, seq_lens, num_processes=2, **kw), host, None, "%s %s (reference build)" % (name, kind))
    hook = _hook(labels, model, alpha, beta, kw["beam"], **opts)
    _same(_res(hook, hook.decode(torch.from_numpy(probs), sl)), host, "%s %s (hook scorer)" % (name, kind))
    x = torch.from_numpy(probs).cuda()
    dev = _res(dec, dec.decode(x, None if sl is None else sl.cuda()))
    _same(host, dev, "%s %s (device entry)" % (name, kind))
    adec = _async(labels, model, alpha, beta, kw["beam"], **opts)
    _same(host, _res(adec, adec.decode(x, None if sl is None else sl.cuda())), "%s %s (async entry)" % (name, kind))


@pytest.mark.parametrize("kind", TWO)
def test_config5_equals_arpa_hook_scorer_and_reference(binaries, kind):
    """config 5 as stated (64 x T=1000 over 29 labels, beam 100, test.arpa, alpha 2.0, beta 1.0) over a binary"""
    probs, _ = c5_text_probs(48, 1000, seed=71)
    probs = torch.cat([probs, ctc_like_probs(16, 1000, 29, seed=72)], 0)
    x = probs.cuda()
    model = binaries[("test.arpa", kind)]
    dec = _dec(L29, model, 2.0, 1.0, 100)
    got = _res(dec, dec.decode(x))
    hook = _hook(L29, model, 2.0, 1.0, 100)
    _same(_res(hook, hook.decode(x)), got, "config 5 %s, hook scorer" % kind)
    if kind == "probing":  # (the same n-grams and values as the ARPA text)
        arpa = _dec(L29, binaries[("test.arpa", "arpa")], 2.0, 1.0, 100)
        _same(_res(arpa, arpa.decode(x)), got, "config 5, probing == ARPA")
    adec = _async(L29, model, 2.0, 1.0, 100)
    _same(got, _res(adec, adec.decode(x)), "config 5 %s, async entry" % kind)
    ref = orc.Reference(L29, model_path=model, alpha=2.0, beta=1.0)
    rows = list(range(0, 64, 4))  # (sampled utterances: the reference build decodes on the CPU)
    want = ref.decode(probs[rows].numpy(), beam=100)
    checked, skipped = compare(want, {k: v[rows] for k, v in got.items()}, None, "config 5 %s, reference build" % kind)
    assert checked >= 10, (checked, skipped)


def _model(binaries, which, kind):
    if which == "word":
        return L29, binaries[("test.arpa", kind)], 2.0, 1.0, 48, c5_text_probs(3, 700, seed=151)[0]
    return LCHAR, binaries[("char_lm", kind)], 1.3, 0.6, 24, ctc_like_probs(3, 700, len(LCHAR), seed=152)


@pytest.mark.parametrize("kind", TWO)
@pytest.mark.parametrize("which", ["word", "char"])
def test_logits_async_graph_and_streaming(binaries, which, kind):
    """fp16 logits; non_blocking equal to the blocking entry; a CUDA graph replayed on new inputs; streaming in uneven
    chunks equal to offline, with each committed prefix a prefix of the final rows"""
    labels, model, alpha, beta, beam, probs = _model(binaries, which, kind)
    what = "%s %s" % (which, kind)
    # fp16 logits against the hook scorer
    x16 = _logits(probs, torch.float16, 153)
    blk = _blocking(labels, model, alpha, beta, beam)
    want16 = _res(blk, blk.decode_logits(x16))
    hook = _hook(labels, model, alpha, beta, beam)
    _same(_res(hook, hook.decode_logits(x16)), want16, what + " f16 logits, hook scorer")
    adec = _async(labels, model, alpha, beta, beam)
    _same(want16, _res(adec, adec.decode_logits(x16)), what + " f16 logits, async entry")
    # a CUDA graph
    x1 = probs.cuda()
    x2 = ctc_like_probs(3, 700, len(labels), seed=154).cuda()
    want1, want2 = _res(blk, blk.decode(x1)), _res(blk, blk.decode(x2))
    _same(_res(hook, hook.decode(x1)), want1, what + " probs, hook scorer")
    static = x1.clone()
    adec.decode(static)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = adec.decode(static)
        nres, flags = adec.last_n_results, adec.last_flags
    for x, want, name in [(x2, want2, "replay 2"), (x1, want1, "replay 1")]:
        static.copy_(x)
        g.replay()
        torch.cuda.synchronize()
        o, s, ts, ln = out
        _same(want, dict(tokens=o.cpu().numpy(), timesteps=ts.cpu().numpy(), scores=s.cpu().numpy(),
                         lens=ln.cpu().numpy(), n_results=nres.cpu().numpy(), ties=flags.cpu().numpy()),
              what + " " + name)
    del g
    # streaming in uneven chunks
    online = ctcdecode_b200.OnlineCTCBeamDecoder(labels, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                                 scorer_provider="device", device_outputs=True, non_blocking=True)
    got, prefixes = _stream_decode(online, x1, 3, False, [0, 50, 187, 188, 488, 700])
    _same(want1, got, what + " streaming")
    for tok, ts, committed in prefixes:
        for b in range(3):
            c = int(committed[b])
            for p in range(int(got["n_results"][b])):
                assert int(got["lens"][b, p]) >= c
                assert np.array_equal(got["tokens"][b, p, :c], tok[b, :c])
                assert np.array_equal(got["timesteps"][b, p, :c], ts[b, :c])


@pytest.mark.parametrize("kind", TWO)
def test_synthetic_order6_model_equals_hook_scorer(binaries, kind):
    """the seeded order-6 model with pruned suffixes (probing collisions, multi-byte trie fields): one batch"""
    model = binaries[("synthetic", kind)]
    words = [w for w in _words(binaries[("synthetic", "arpa")]) if w not in ("<s>", "</s>", "<unk>")]
    rng = random.Random(61)
    texts = [" ".join(rng.choice(words) for _ in range(12)) for _ in range(12)]
    probs = torch.cat([text_probs(texts, L29, 400, seed=62), ctc_like_probs(4, 400, 29, seed=63)], 0)
    dec = _dec(L29, model, 1.2, 0.4, 64)
    assert dec.max_order() == 6
    got = _res(dec, dec.decode(probs.cuda()))
    hook = _hook(L29, model, 1.2, 0.4, 64)
    _same(_res(hook, hook.decode(probs.cuda())), got, "synthetic order 6 %s" % kind)


def test_refused_binary_is_followed_by_exact_decodes(binaries, tmp_path):
    model = binaries[("test.arpa", "probing")]
    probs = text_probs(TEXTS, L29, 100, seed=121)
    x = probs.cuda()
    dec = _dec(L29, model, 1.0, 0.5, 16)
    hook = _hook(L29, model, 1.0, 0.5, 16)
    want = _res(hook, hook.decode(probs))
    _same(want, _res(dec, dec.decode(x)), "before")
    data = bytearray(open(model, "rb").read())
    data[96] = 1  # REST_PROBING
    bad = tmp_path / "rest.binary"
    bad.write_bytes(bytes(data))
    with pytest.raises(_native.NativeError, match="error -2: .*KenLM binary.*REST_PROBING"):
        _dec(L29, str(bad), 1.0, 0.5, 16)
    _same(want, _res(dec, dec.decode(x)), "after a refused binary")
    fresh = _dec(L29, model, 1.0, 0.5, 16)
    _same(want, _res(fresh, fresh.decode(x)), "a fresh scorer after the refusal")
