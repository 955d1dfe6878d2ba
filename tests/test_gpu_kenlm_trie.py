"""KenLM trie files searched in place in HBM (-m gpu): the wide order-5 model of tests/test_kenlm_trie_inplace.py (17-bit
word ids, nodes of thousands of children, Bhiksha-compressed pointers) in its four trie types.  The blocking, device,
asynchronous and streaming decodes must equal, bit for bit, the hook scorer over the same file (the reference's Scorer
over KenLM); the blocking entry also equals the reference build.  Each runs under the default launch plan and with
128-thread beam CTAs."""
import os
import random

import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200.scorer import ArpaScorer
from ctcdecode_b200.synth import ctc_like_probs, text_probs
from oracle import oracle as orc
from tests.parity import compare
from tests.test_gpu_lm_async import _async, _stream_decode
from tests.test_gpu_ngram_scorer import _dec, _hook, _res, _same
from tests.test_kenlm_binary import BUILD_BINARY, L29
from tests.test_kenlm_trie_inplace import TRIES, wide  # noqa: F401 (a fixture)

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)"),
    pytest.mark.skipif(not os.path.exists(orc.PROVIDER), reason="scorer provider (make -C oracle provider) not built"),
    pytest.mark.skipif(not os.path.exists(BUILD_BINARY),
                       reason="build_binary (make -C oracle -f build_binary.mk build_binary) not built"),
]


@pytest.mark.parametrize("nt", [None, 128])
@pytest.mark.parametrize("kind", TRIES)
def test_wide_trie_through_every_entry(wide, kind, nt, monkeypatch):
    if nt:
        monkeypatch.setenv("CTCDEC_NT", str(nt))
    arpa, grams, paths = wide
    model = paths[kind]
    rng = random.Random(91)
    texts = [" ".join(" ".join(rng.choice(grams[4])) for _ in range(3)) for _ in range(6)]
    probs = torch.cat([text_probs(texts, L29, 300, seed=92), ctc_like_probs(2, 300, 29, seed=93)], 0)
    alpha, beta, beam = 1.4, 0.6, 48
    what = "wide %s nt=%s" % (kind, nt)
    assert ArpaScorer(L29, model, alpha, beta).table_bytes() <= os.path.getsize(model)

    dec = _dec(L29, model, alpha, beta, beam)
    want = _res(dec, dec.decode(probs))
    hook = _hook(L29, model, alpha, beta, beam)
    _same(_res(hook, hook.decode(probs)), want, what + " hook scorer")
    rows = list(range(0, 8, 2))
    ref = orc.Reference(L29, model_path=model, alpha=alpha, beta=beta).decode(probs[rows].numpy(), beam=beam)
    checked, _ = compare(ref, {k: v[rows] for k, v in want.items()}, None, what + " reference build")
    assert checked >= 3
    x = probs.cuda()
    _same(want, _res(dec, dec.decode(x)), what + " device entry")
    adec = _async(L29, model, alpha, beta, beam)
    _same(want, _res(adec, adec.decode(x)), what + " async entry")
    online = ctcdecode_b200.OnlineCTCBeamDecoder(L29, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                                 scorer_provider="device", device_outputs=True, non_blocking=True)
    got, _ = _stream_decode(online, x, 8, False, [0, 37, 38, 150, 299, 300])
    _same(want, got, what + " streaming")
