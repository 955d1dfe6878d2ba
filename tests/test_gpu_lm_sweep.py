"""A sweep of the LM weights on the GPU (-m gpu): CTCBeamDecoder.decode_sweep / ctcdec_decode_batch_lm_sweep_async.
Slice p of every output must equal, bit for bit, the asynchronous device decode of the same batch after
reset_params(alphas[p], betas[p])."""
import os

import numpy as np
import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200.synth import ctc_like_probs, text_probs
from oracle import oracle as orc
from tests import golden_util
from tests.parity import compare
from tests.test_gpu_ngram_scorer import _logits, _res, _same
from tests.test_lm import c5_text_probs

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)"),
]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
REF_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
BUILD_BINARY = os.path.join(ROOT, "oracle", "_ref", "build_binary")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]
TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran"]
PAIRS = [(0.0, 0.0), (1.5, -0.8), (0.7, 4.0), (2.25, 1.1)]


def _async(labels, model, alpha, beta, beam, **kw):
    dec = ctcdecode_b200.CTCBeamDecoder(labels, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                        scorer_provider="device", device_outputs=True, non_blocking=True, **kw)
    dec.ab = (alpha, beta)
    return dec


def _slice(dec, out, p):
    o, s, ts, ln = out
    return dict(tokens=o[p].cpu().numpy(), timesteps=ts[p].cpu().numpy(), scores=s[p].cpu().numpy(),
                lens=ln[p].cpu().numpy(), n_results=dec.last_n_results[p].cpu().numpy(),
                ties=dec.last_flags[p].cpu().numpy())


def _one_by_one(dec, x, pairs, sl=None, logits=False):
    """the baseline: one asynchronous decode per pair after reset_params (the decoder's own pair, dec.ab, restored
    after)"""
    a0, b0 = dec.ab
    out = []
    for a, b in pairs:
        dec.reset_params(a, b)
        out.append(_res(dec, dec.decode_logits(x, sl) if logits else dec.decode(x, sl)))
    dec.reset_params(a0, b0)
    return out


def _check(dec, x, pairs, sl=None, logits=False, name=""):
    want = _one_by_one(dec, x, pairs, sl, logits)
    out = dec.decode_sweep(x, [a for a, _ in pairs], [b for _, b in pairs], seq_lens=sl, logits=logits)
    assert out[0].shape[:2] == (len(pairs), x.shape[0]) and dec.last_flags.shape == (len(pairs), x.shape[0])
    got = [_slice(dec, out, p) for p in range(len(pairs))]
    for p in range(len(pairs)):
        _same(want[p], got[p], "%s pair %d" % (name, p))
    return got


@pytest.mark.parametrize("name", golden_util.names(lm=True) + golden_util.names_char())
def test_fixtures_equal_reset_params_decodes(name):
    probs, seq_lens, kw, gold, alpha, beta = golden_util.load_lm(name)
    labels, model = (LCHAR, CHAR_LM) if name.startswith("lmchar_") else (L29, TINY)
    dec = _async(labels, model, alpha, beta, kw["beam"], cutoff_top_n=kw["cutoff_top_n"],
                 cutoff_prob=kw["cutoff_prob"], log_probs_input=kw["log_input"])
    x = torch.from_numpy(probs).cuda()
    sl = None if seq_lens is None else torch.as_tensor(seq_lens).cuda()
    got = _check(dec, x, PAIRS + [(alpha, beta)], sl, name=name)
    if float(np.float32(alpha)) == alpha and float(np.float32(beta)) == beta:
        # (the fixture was made with a scorer constructed with the unrounded doubles: a sweep rounds them as
        # reset_params does, so the two agree only where the rounding changes nothing)
        compare(gold, got[-1], None, name + " (fixture)")


@pytest.mark.parametrize("model", ["tiny", "char"])
def test_fp16_logits(model):
    labels, path = (L29, TINY) if model == "tiny" else (LCHAR, CHAR_LM)
    probs = text_probs(TEXTS * 2, L29, 150, seed=81) if model == "tiny" else ctc_like_probs(6, 120, len(LCHAR), seed=82)
    x = _logits(probs, torch.float16, 83)
    sl = torch.tensor([150, 0, 1, 77, 149, 120], dtype=torch.int32).clamp(max=probs.shape[1]).cuda()
    _check(_async(labels, path, 1.0, 0.5, 24), x, PAIRS, sl, logits=True, name="fp16 " + model)


def test_cpu_input_and_a_single_pair():
    probs = text_probs(TEXTS, L29, 100, seed=91)
    dec = _async(L29, TINY, 1.2, 0.3, 16)
    want = _one_by_one(dec, probs.cuda(), [(0.9, -0.4)])
    out = dec.decode_sweep(probs, [0.9], [-0.4])  # CPU input: uploaded, the call waits, CPU results
    assert not out[0].is_cuda and out[0].shape == (1, 3, 16, 100) and not dec.last_flags.is_cuda
    _same(want[0], _slice(dec, out, 0), "CPU input, P = 1")


def test_config5_p8_equals_async_decodes_and_reference():
    """config 5 (64 x T=1000, 29 labels, beam 100, test.arpa) at P = 8: 512 beam CTAs, two waves"""
    probs, _ = c5_text_probs(48, 1000, seed=71)
    probs = torch.cat([probs, ctc_like_probs(16, 1000, 29, seed=72)], 0)
    pairs = [(2.0, 1.0), (0.0, 0.0), (0.5, -1.0), (1.0, 0.5), (1.5, 2.0), (2.5, 1.5), (3.0, -0.5), (2.0, 6.0)]
    dec = _async(L29, REF_ARPA, 2.0, 1.0, 100)
    got = _check(dec, probs.cuda(), pairs, name="config 5")
    ref = orc.Reference(L29, model_path=REF_ARPA, alpha=2.0, beta=1.0)
    for p in (0, 2, 7):
        ref.lib.ref_scorer_reset_params(ref.scorer, *pairs[p])
        checked, skipped = compare(ref.decode(probs.numpy(), beam=100), got[p], None, "config 5 pair %d, reference" % p)
        assert checked >= 40, (p, checked, skipped)


@pytest.mark.skipif(not os.path.exists(BUILD_BINARY), reason="oracle/_ref/build_binary not built")
def test_kenlm_trie_equals_its_arpa_text(tmp_path):
    from tests.test_kenlm_binary import build_binary
    trie = build_binary(REF_ARPA, tmp_path, "trie")
    x = ctc_like_probs(8, 200, 29, seed=95).cuda()
    a = _async(L29, REF_ARPA, 2.0, 1.0, 32)
    t = _async(L29, trie, 2.0, 1.0, 32)
    oa = a.decode_sweep(x, [a_ for a_, _ in PAIRS], [b for _, b in PAIRS])
    ot = t.decode_sweep(x, [a_ for a_, _ in PAIRS], [b for _, b in PAIRS])
    for p in range(len(PAIRS)):
        _same(_slice(a, oa, p), _slice(t, ot, p), "trie pair %d" % p)


def test_graph_replays_the_captured_pairs_on_new_input():
    x1 = text_probs(TEXTS * 2, L29, 120, seed=201).cuda()
    x2 = ctc_like_probs(6, 120, 29, seed=202).cuda()
    dec = _async(L29, TINY, 1.5, 0.8, 32)
    want1, want2 = _one_by_one(dec, x1, PAIRS), _one_by_one(dec, x2, PAIRS)
    al, be = [a for a, _ in PAIRS], [b for _, b in PAIRS]
    static = x1.clone()
    dec.decode_sweep(static, al, be)  # outside the capture: tables uploaded, kernel limits raised, workspace sized
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = dec.decode_sweep(static, al, be)
        nres, flags = dec.last_n_results, dec.last_flags
    for x, want, name in [(x1, want1, "replay 1"), (x2, want2, "replay 2")]:
        static.copy_(x)
        g.replay()
        torch.cuda.synchronize()
        for p in range(len(PAIRS)):
            o, s, ts, ln = out
            got = dict(tokens=o[p].cpu().numpy(), timesteps=ts[p].cpu().numpy(), scores=s[p].cpu().numpy(),
                       lens=ln[p].cpu().numpy(), n_results=nres[p].cpu().numpy(), ties=flags[p].cpu().numpy())
            _same(want[p], got, "%s pair %d" % (name, p))


def test_the_decoders_own_weights_are_unchanged():
    x = text_probs(TEXTS, L29, 120, seed=221).cuda()
    dec = _async(L29, TINY, 1.0, 0.5, 24)
    before = _res(dec, dec.decode(x))
    dec.decode_sweep(x, [2.5, 0.0], [-0.5, 3.0])
    _same(before, _res(dec, dec.decode(x)), "decode after a sweep")


def test_refusals():
    x = text_probs(TEXTS, L29, 60, seed=5).cuda()
    with pytest.raises(ValueError, match="scorer_provider"):
        ctcdecode_b200.CTCBeamDecoder(L29, beam_width=8, device_outputs=True).decode_sweep(x, [1.0], [0.5])
    if os.path.exists(orc.PROVIDER):  # a hook scorer
        hook = ctcdecode_b200.CTCBeamDecoder(L29, model_path=TINY, alpha=1.0, beta=0.5, beam_width=8,
                                             scorer_provider=orc.PROVIDER)
        with pytest.raises(ValueError, match="scorer_provider"):
            hook.decode_sweep(x, [1.0], [0.5])
    dec = _async(L29, TINY, 1.0, 0.5, 8)
    with pytest.raises(ValueError, match="equal length"):
        dec.decode_sweep(x, [1.0, 2.0], [0.5])
    with pytest.raises(ValueError, match="non-empty"):
        dec.decode_sweep(x, [], [])
