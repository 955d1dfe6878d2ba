"""A decode over several language models on the GPU (-m gpu): CTCBeamDecoder.decode_mixed /
ctcdec_decode_batch_lm_mixed_async.  Utterance b must equal, bit for bit and flags included, the asynchronous device
decode of its model's sub-batch, and the reference build's decode with that model and weights."""
import os

import numpy as np
import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200 import _native
from ctcdecode_b200.synth import ctc_like_probs
from oracle import oracle as orc
from tests.parity import compare
from tests.test_gpu_ngram_scorer import _logits, _res, _same
from tests.test_lm import c5_text_probs
from tests.test_lm_mixed_emulation import _char_bigram

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


def _dec(labels, model, alpha, beta, beam, **kw):
    d = ctcdecode_b200.CTCBeamDecoder(labels, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                      scorer_provider="device", device_outputs=True, non_blocking=True, **kw)
    d.spec = (model, alpha, beta)
    return d


@pytest.fixture(scope="module")
def word_models(tmp_path_factory):
    """test.arpa at two weight pairs, tiny_lm, and a trie file of test.arpa (its ARPA text without build_binary)"""
    trie = REF_ARPA
    if os.path.exists(BUILD_BINARY):
        from tests.test_kenlm_binary import build_binary
        trie = build_binary(REF_ARPA, tmp_path_factory.mktemp("mixed"), "trie")
    return [(REF_ARPA, 1.5, 0.8), (REF_ARPA, 0.5, 2.0), (TINY, 2.0, -1.0), (trie, 1.0, 1.0)]


def _rows(d, rows):
    return {k: v[rows] for k, v in d.items()}


def _lm_index(B, S, seed):
    g = np.random.default_rng(seed)
    idx = g.integers(0, S, B).astype(np.int32)
    idx[:S] = np.arange(S)   # every model takes an utterance
    return idx


def _check_against_sub_batches(decs, x, lm_index, sl, logits=False, name=""):
    got = _res(decs[0], decs[0].decode_mixed(x, torch.from_numpy(lm_index), decs, sl, logits=logits))
    for s, d in enumerate(decs):
        rows = np.nonzero(lm_index == s)[0]
        r = torch.from_numpy(rows).to(x.device)
        xs, ss = x.index_select(0, r), (sl.index_select(0, r.to(sl.device)) if sl is not None else None)
        want = _res(d, d.decode_logits(xs, ss) if logits else d.decode(xs.cuda(), ss.cuda() if ss is not None else None))
        _same(want, _rows(got, rows), "%s model %d" % (name, s))
    return got


@pytest.mark.parametrize("inp", ["cuda_f32", "cpu_f32", "cuda_f16_logits"])
def test_config5_word_models_against_per_model_decodes(word_models, inp):
    """config-5 shape (64 x 1000 x 29, beam 100), four scorers, a random lm_index, ragged lengths including 0"""
    probs, _ = c5_text_probs(64, 1000, seed=71)
    decs = [_dec(L29, m, a, b, 100) for m, a, b in word_models]
    sl = torch.randint(1, 1001, (64,), generator=torch.Generator().manual_seed(3), dtype=torch.int32)
    sl[5], sl[6], sl[7] = 0, 1000, 1
    lm_index = _lm_index(64, len(decs), seed=9)
    if inp == "cuda_f16_logits":
        _check_against_sub_batches(decs, _logits(probs, torch.float16, 5), lm_index, sl.cuda(), logits=True, name=inp)
    elif inp == "cuda_f32":
        _check_against_sub_batches(decs, probs.cuda(), lm_index, sl.cuda(), name=inp)
    else:
        _check_against_sub_batches(decs, probs, lm_index, sl, name=inp)


@pytest.mark.parametrize("inp", ["cuda_f32", "cpu_f32", "cuda_f16_logits"])
def test_char_models_against_per_model_decodes(tmp_path, inp):
    """char_lm beside a generated character bigram model"""
    other = _char_bigram(str(tmp_path / "char_bigram.arpa"))
    decs = [_dec(LCHAR, CHAR_LM, 1.0, 0.5, 24), _dec(LCHAR, other, 2.0, -0.5, 24), _dec(LCHAR, CHAR_LM, 0.3, 2.0, 24)]
    probs = ctc_like_probs(40, 300, len(LCHAR), seed=35)
    sl = torch.randint(0, 301, (40,), generator=torch.Generator().manual_seed(4), dtype=torch.int32)
    sl[3] = 0
    idx = _lm_index(40, 3, seed=2)
    if inp == "cuda_f16_logits":
        _check_against_sub_batches(decs, _logits(probs, torch.float16, 6), idx, sl.cuda(), logits=True, name=inp)
    elif inp == "cuda_f32":
        _check_against_sub_batches(decs, probs.cuda(), idx, sl.cuda(), name=inp)
    else:
        _check_against_sub_batches(decs, probs, idx, sl, name=inp)


def test_against_the_reference_build(word_models):
    """each utterance against oracle.Reference with its model and weights, through tests/parity.py's tie rules"""
    probs, _ = c5_text_probs(16, 400, seed=5)
    decs = [_dec(L29, m, a, b, 32) for m, a, b in word_models[:3]]
    lm_index = _lm_index(16, 3, seed=1)
    sl = torch.tensor([400, 0, 1, 250] + [400 - 9 * i for i in range(12)], dtype=torch.int32)
    got = _res(decs[0], decs[0].decode_mixed(probs.cuda(), torch.from_numpy(lm_index), decs, sl.cuda()))
    for s, (m, a, b) in enumerate(word_models[:3]):
        rows = np.nonzero(lm_index == s)[0]
        ref = orc.Reference(L29, model_path=m, alpha=a, beta=b)
        want = ref.decode(probs.numpy()[rows], sl.numpy()[rows], num_processes=2, beam=32)
        compare(want, _rows(got, rows), None, "model %d" % s)


def test_graph_replay(word_models):
    """captured after one decode outside the capture, a replay gives the uncaptured results"""
    probs, _ = c5_text_probs(24, 300, seed=13)
    decs = [_dec(L29, m, a, b, 32) for m, a, b in word_models]
    lm_index = torch.from_numpy(_lm_index(24, len(decs), seed=4))
    x = probs.cuda()
    want = _res(decs[0], decs[0].decode_mixed(x, lm_index, decs))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        decs[0].decode_mixed(x, lm_index, decs)   # (workspace and outputs allocated on the capture stream's pool)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            out = decs[0].decode_mixed(x, lm_index, decs)
    g.replay()
    torch.cuda.synchronize()
    _same(want, _res(decs[0], out), "replay")


def test_refusals(word_models):
    probs = ctc_like_probs(2, 20, 29, seed=1).cuda()
    decs = [_dec(L29, m, a, b, 8) for m, a, b in word_models[:2]]
    with pytest.raises(ValueError, match="scorer_provider"):
        decs[0].decode_mixed(probs, [0, 1], decs + [ctcdecode_b200.CTCBeamDecoder(L29, beam_width=8)])
    with pytest.raises(_native.NativeError, match="outside"):
        decs[0].decode_mixed(probs, [0, 2], decs)
    ch, wd = _dec(LCHAR, CHAR_LM, 1.0, 1.0, 8), _dec(LCHAR, TINY, 1.0, 1.0, 8)   # (tiny_lm: word-based over LCHAR)
    with pytest.raises(_native.NativeError, match="both word-based or both character-based"):
        ch.decode_mixed(ctc_like_probs(2, 20, len(LCHAR), seed=1).cuda(), [0, 1], [ch, wd])
    with pytest.raises(ValueError, match="other labels"):
        decs[0].decode_mixed(probs, [0, 1], [decs[0], ch])
    with pytest.raises(_native.NativeError, match="1 to 16"):
        decs[0].decode_mixed(probs, [0, 1], decs * 9)
    other = list(L29)
    other[5] = "E"
    with pytest.raises(ValueError, match="other labels"):
        decs[0].decode_mixed(probs, [0, 1], [decs[0], _dec(other, REF_ARPA, 1.0, 1.0, 8)])


# ---- streams of different models in one call --------------------------------------------------------------------
STREAM_MODELS = [(REF_ARPA, 1.5, 0.8), (TINY, 2.0, -1.0)]


def _online(labels, model, alpha, beta, beam, device_entry, **kw):
    extra = dict(device_outputs=True, non_blocking=True) if device_entry else {}
    return ctcdecode_b200.OnlineCTCBeamDecoder(labels, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                               scorer_provider="device", **extra, **kw)


def _stream_row(out, dec, i):
    """stream i of one decode's results as a one-utterance dict (CPU numpy)"""
    o, sc, ts, ln = (t.cpu() for t in out)
    return dict(tokens=o[i:i + 1].numpy(), timesteps=ts[i:i + 1].numpy(), scores=sc[i:i + 1].numpy(),
                lens=ln[i:i + 1].numpy(), n_results=dec.last_n_results.cpu()[i:i + 1].numpy(),
                ties=dec.last_flags.cpu()[i:i + 1].numpy())


@pytest.mark.parametrize("entry", ["host", "device"])
def test_streams_of_two_models_against_the_reference(entry):
    """states of two device-scorer decoders in one OnlineCTCBeamDecoder.decode call per chunk, against states of two
    reference decoders in one decode_with_states call per chunk (and each stream's offline reference decode); CPU
    chunks go through the host entry, CUDA chunks with non_blocking=True through the device entry; the streams reach
    eos at different chunks"""
    beam, F = 16, 30
    decs = [_online(L29, m, a, b, beam, entry == "device") for m, a, b in STREAM_MODELS]
    refs = [orc.Reference(L29, model_path=m, alpha=a, beta=b) for m, a, b in STREAM_MODELS]
    probs, _ = c5_text_probs(5, 3 * F, seed=8)
    model_of = [0, 1, 1, 0, 1]
    last = [1, 2, 0, 2, 2]          # the chunk at which each stream reaches eos
    st = [ctcdecode_b200.DecoderState(decs[m]) for m in model_of]
    rst = [refs[m].state_new(beam) for m in model_of]
    try:
        for c in range(3):
            live = [s for s in range(5) if last[s] >= c]
            chunk = probs[live, F * c:F * (c + 1)].contiguous()
            eos = [last[s] == c for s in live]
            out = decs[0].decode(chunk.cuda() if entry == "device" else chunk, [st[s] for s in live], eos)
            want = refs[0].decode_with_states(chunk.numpy(), [rst[s] for s in live], eos, beam, max_len=4 * F)
            for i, s in enumerate(live):
                if not eos[i]:
                    continue
                got = _stream_row(out, decs[0], i)
                m, a, b = STREAM_MODELS[model_of[s]]
                off = refs[model_of[s]].decode(probs[s:s + 1, :F * (c + 1)].numpy(), None, num_processes=1, beam=beam)
                n = got["tokens"].shape[2]
                want_s = dict(tokens=want["tokens"][i:i + 1, :, :n], timesteps=want["timesteps"][i:i + 1, :, :n],
                              scores=want["scores"][i:i + 1], lens=want["lens"][i:i + 1], n_results=off["n_results"])
                name = "%s stream %d (model %d, eos at chunk %d)" % (entry, s, model_of[s], c)
                compare(want_s, got, None, name + " vs reference streaming")
                compare(off, got, None, name + " vs reference offline")
    finally:
        for r in rst:
            refs[0].state_free(r)


def test_stream_refusals():
    """states that cannot share a call, through OnlineCTCBeamDecoder.decode (host and device entries)"""
    probs = ctc_like_probs(2, 4, 29, seed=1)
    a = _online(L29, REF_ARPA, 1.0, 1.0, 8, True)
    b = _online(L29, TINY, 1.0, 1.0, 8, True)

    def pair(x, y):
        return [ctcdecode_b200.DecoderState(x), ctcdecode_b200.DecoderState(y)]

    cases = [
        (_online(L29, TINY, 1.0, 1.0, 8, True, cutoff_top_n=5), "same decoder configuration"),
        (ctcdecode_b200.OnlineCTCBeamDecoder(L29, beam_width=8, device_outputs=True, non_blocking=True),
         "without one"),
        (_online(LCHAR[:1] + L29[1:], CHAR_LM, 1.0, 1.0, 8, True), "different labels|character-based"),
    ]
    other = list(L29)
    other[5] = "E"
    cases.append((_online(other, TINY, 1.0, 1.0, 8, True), "different labels"))
    for x in (probs, probs.cuda()):
        assert a.decode(x, pair(a, b), [True, True])[0].shape[0] == 2    # two models: accepted
        for dec, msg in cases:
            with pytest.raises(_native.NativeError, match=msg):
                a.decode(x, pair(a, dec), [False, False])


def test_stream_states_workspace():
    """the states-aware size: ctcdec_stream_workspace_bytes for states of one scorer (or none), plus the streams'
    slot indices and one 256-byte slot per scorer for states of several"""
    import ctypes
    lib = _native.load()
    a = _online(L29, REF_ARPA, 1.0, 1.0, 8, True)
    b = _online(L29, TINY, 1.0, 1.0, 8, True)
    plain = ctcdecode_b200.OnlineCTCBeamDecoder(L29, beam_width=8)
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    for B, T in ((1, 1), (3, 40), (300, 7)):
        cfg = _native.Config(29, 8, 0, 0, 40, 1.0)
        one = ctypes.c_size_t(0)
        assert lib.ctcdec_stream_workspace_bytes(ctypes.byref(cfg), B, T, ctypes.byref(one)) == 0
        for decs, extra in (([a], 0), ([plain], 0), ([a, b], al(B) + al(2 * 256))):
            if len(decs) > B:
                continue
            st = [ctcdecode_b200.DecoderState(decs[i % len(decs)]) for i in range(B)]
            h = (ctypes.c_void_p * B)(*[s.state for s in st])
            n = ctypes.c_size_t(0)
            assert lib.ctcdec_stream_states_workspace_bytes(h, B, T, ctypes.byref(n)) == 0
            assert n.value == one.value + extra, (B, T, len(decs))
