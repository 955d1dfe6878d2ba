"""The scorer path on the H100 (-m gpu) where LM terms are positive: alpha < 0 on word and character models, and a word
model whose backoff weights lift conditional log-probs above 0.  The beam kernel's radix histogram must still hold
every key (beam_program.cuh, the scorer branch of the frame head), so every entry point equals the reference build."""
import os

import numpy as np
import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200.synth import ctc_like_probs, text_probs
from oracle import oracle as orc
from tests.parity import compare
from tests.test_gpu_lm_async import _stream_decode
from tests.test_gpu_lm_sweep import _check, _slice
from tests.test_gpu_ngram_scorer import _hook, _logits, _res, _same
from tests.test_lm import c5_text_probs
from tests.test_lm_weights_emulation import BACKOFF_TEXTS, POSITIVE_BACKOFF_ARPA, SWEEP_PAIRS

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref (the reference build) not built"),
]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
REF_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]


@pytest.fixture(params=["word", "char", "backoff"])
def model(request, tmp_path):
    """(labels, model path, alpha, beta, beam, probs, seq_lens)"""
    if request.param == "word":
        probs = ctc_like_probs(4, 150, 29, seed=5)
        return L29, REF_ARPA, -2.0, 1.0, 32, probs, torch.tensor([150, 0, 1, 97], dtype=torch.int32)
    if request.param == "char":
        probs = ctc_like_probs(4, 120, len(LCHAR), seed=6)
        return LCHAR, CHAR_LM, -2.0, 1.0, 24, probs, torch.tensor([120, 1, 0, 64], dtype=torch.int32)
    path = tmp_path / "positive_backoff.arpa"
    path.write_text(POSITIVE_BACKOFF_ARPA)
    probs = text_probs(BACKOFF_TEXTS, L29, 120, seed=41)
    return L29, str(path), 1.5, 0.5, 32, probs, torch.tensor([120, 77, 1], dtype=torch.int32)


def _dec(labels, path, alpha, beta, beam, **kw):
    return ctcdecode_b200.CTCBeamDecoder(labels, model_path=path, alpha=alpha, beta=beta, beam_width=beam,
                                         scorer_provider="device", **kw)


def test_host_device_and_non_blocking_entries(model):
    labels, path, alpha, beta, beam, probs, sl = model
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    want = ref.decode(probs.numpy(), sl.numpy(), beam=beam, num_processes=2)
    dec = _dec(labels, path, alpha, beta, beam)
    host = _res(dec, dec.decode(probs, sl))
    compare(want, host, None, "host entry")
    _same(host, _res(dec, dec.decode(probs.cuda(), sl.cuda())), "device entry")
    nb = _dec(labels, path, alpha, beta, beam, device_outputs=True, non_blocking=True)
    _same(host, _res(nb, nb.decode(probs.cuda(), sl.cuda())), "non-blocking entry")


def test_f16_logits(model):
    labels, path, alpha, beta, beam, probs, sl = model
    x = _logits(probs, torch.float16, 7)
    dec = _dec(labels, path, alpha, beta, beam)
    *res, lsm = dec.decode_logits(x, sl, return_log_probs=True)
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    want = ref.decode(lsm.cpu().numpy(), sl.numpy(), beam=beam, log_input=True, num_processes=2)
    compare(want, _res(dec, res), None, "f16 logits")


def test_sweep_mixing_signs(model):
    """each CTA bounds its keys with its own pair: every slice equals the decode after reset_params"""
    labels, path, alpha, beta, beam, probs, sl = model
    dec = _dec(labels, path, alpha, beta, beam, device_outputs=True, non_blocking=True)
    dec.ab = (alpha, beta)
    got = _check(dec, probs.cuda(), SWEEP_PAIRS + [(alpha, beta)], sl.cuda(), name="sweep")
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    compare(ref.decode(probs.numpy(), sl.numpy(), beam=beam, num_processes=2), got[-1], None, "sweep, own pair")


def test_streaming_chunks_equal_offline(model):
    labels, path, alpha, beta, beam, probs, sl = model
    off = _dec(labels, path, alpha, beta, beam)
    want = _res(off, off.decode(probs.cuda()))
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(labels, model_path=path, alpha=alpha, beta=beta, beam_width=beam,
                                              scorer_provider="device", device_outputs=True, non_blocking=True)
    got, _ = _stream_decode(dec, probs.cuda(), probs.shape[0], False, [0, 7, 50, 51, probs.shape[1]])
    _same(want, got, "streaming")


@pytest.mark.skipif(not os.path.exists(orc.PROVIDER), reason="scorer provider (make -C oracle provider) not built")
def test_hook_scorer(model):
    """the reference's Scorer behind the host hook: the kernel sees only the terms, not alpha"""
    labels, path, alpha, beta, beam, probs, sl = model
    hook = _hook(labels, path, alpha, beta, beam)
    got = _res(hook, hook.decode(probs, sl))
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    compare(ref.decode(probs.numpy(), sl.numpy(), beam=beam, num_processes=2), got, None, "hook scorer")
    dec = _dec(labels, path, alpha, beta, beam)
    _same(_res(dec, dec.decode(probs, sl)), got, "hook scorer vs device scorer")


def test_config5_shape_at_negative_alpha():
    """config 5's shape: 64 x T=1000 over 29 labels, beam 100, test.arpa, at alpha -1, beta 1"""
    probs, _ = c5_text_probs(48, 1000, seed=71)
    probs = torch.cat([probs, ctc_like_probs(16, 1000, 29, seed=72)], 0)
    dec = _dec(L29, REF_ARPA, -1.0, 1.0, 100)
    got = _res(dec, dec.decode(probs.cuda()))
    ref = orc.Reference(L29, model_path=REF_ARPA, alpha=-1.0, beta=1.0)
    checked, skipped = compare(ref.decode(probs.numpy(), beam=100), got, None, "config 5 shape, alpha -1")
    assert checked >= 40, (checked, skipped)
    sw = _dec(L29, REF_ARPA, -1.0, 1.0, 100, device_outputs=True, non_blocking=True)
    out = sw.decode_sweep(probs.cuda(), [-1.0, 2.0], [1.0, 1.0])
    _same(got, _slice(sw, out, 0), "config 5 shape, sweep slice")
