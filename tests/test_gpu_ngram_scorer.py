"""The library's own ARPA scorer on the H100 (-m gpu): scorer_provider="device" builds it from the model file, and the beam
kernel computes its LM terms in the CTA (no per-frame host handshake).  Every decode must equal, bit for bit, the
decode with the reference's Scorer behind the hook (the provider library) and the reference build itself."""
import ctypes
import os
import threading

import numpy as np
import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200 import _native
from ctcdecode_b200.synth import ctc_like_probs, text_probs
from oracle import oracle as orc
from tests import golden_util
from tests.parity import compare
from tests.test_lm import c5_text_probs

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)"),
    pytest.mark.skipif(not os.path.exists(orc.PROVIDER), reason="scorer provider (make -C oracle provider) not built"),
]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
REF_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]
TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran"]


def _dec(labels, model, alpha, beta, beam, provider="device", **kw):
    return ctcdecode_b200.CTCBeamDecoder(labels, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                         scorer_provider=provider, **kw)


def _hook(labels, model, alpha, beta, beam, **kw):
    return _dec(labels, model, alpha, beta, beam, provider=orc.PROVIDER, **kw)


def _res(dec, out):
    o, s, ts, ln = out
    return dict(tokens=o.cpu().numpy(), timesteps=ts.cpu().numpy(), scores=s.cpu().numpy(), lens=ln.cpu().numpy(),
                n_results=dec.last_n_results.cpu().numpy(), ties=dec.last_flags.cpu().numpy())


def _same(want, got, name):
    """bit for bit: n_results, flags, and for every row p < n_results the score bits, the length, tokens and timesteps"""
    assert np.array_equal(want["n_results"], got["n_results"]), name
    assert np.array_equal(want["ties"], got["ties"]), name
    for b in range(want["n_results"].shape[0]):
        n = int(want["n_results"][b])
        assert np.array_equal(want["scores"][b, :n].view(np.int32), got["scores"][b, :n].view(np.int32)), (name, b)
        assert np.array_equal(want["lens"][b, :n], got["lens"][b, :n]), (name, b)
        for p in range(n):
            L = int(want["lens"][b, p])
            assert np.array_equal(want["tokens"][b, p, :L], got["tokens"][b, p, :L]), (name, b, p)
            assert np.array_equal(want["timesteps"][b, p, :L], got["timesteps"][b, p, :L]), (name, b, p)


def _logits(probs, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = probs.clamp_min(1e-20).log() * 1.25 + 0.3 * torch.randn(probs.shape, generator=g)
    return x.to(dtype).cuda()


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", golden_util.names(lm=True) + golden_util.names_char())
def test_fixtures_through_host_and_device_entries(name):
    probs, seq_lens, kw, gold, alpha, beta = golden_util.load_lm(name)
    labels, model = (LCHAR, CHAR_LM) if name.startswith("lmchar_") else (L29, TINY)
    opts = dict(cutoff_top_n=kw["cutoff_top_n"], cutoff_prob=kw["cutoff_prob"], log_probs_input=kw["log_input"])
    dec = _dec(labels, model, alpha, beta, kw["beam"], **opts)
    sl = None if seq_lens is None else torch.as_tensor(seq_lens)
    host = _res(dec, dec.decode(torch.from_numpy(probs), sl))
    compare(gold, host, None, name + " (host entry)")
    dev = _res(dec, dec.decode(torch.from_numpy(probs).cuda(), None if sl is None else sl.cuda()))
    _same(host, dev, name + " (device entry)")
    hook = _hook(labels, model, alpha, beta, kw["beam"], **opts)
    _same(_res(hook, hook.decode(torch.from_numpy(probs), sl)), host, name + " (hook scorer)")


@pytest.mark.parametrize("model", ["tiny", "char"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
def test_logits_match_reference(dtype, model):
    if model == "tiny":
        labels, path, alpha, beta, beam = L29, TINY, 1.5, 0.7, 32
        probs = text_probs(TEXTS * 2, L29, 150, seed=81)
    else:
        labels, path, alpha, beta, beam = LCHAR, CHAR_LM, 1.3, 0.6, 24
        probs = ctc_like_probs(6, 120, len(LCHAR), seed=82)
    x = _logits(probs, dtype, 83)
    sl = torch.tensor([150, 0, 1, 77, 149, 120], dtype=torch.int32).clamp(max=probs.shape[1])
    dec = _dec(labels, path, alpha, beta, beam)
    *res, lsm = dec.decode_logits(x, sl, return_log_probs=True)
    got = _res(dec, res)
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    want = ref.decode(lsm.cpu().numpy(), sl.numpy(), beam=beam, log_input=True, num_processes=2)
    compare(want, got, None, "logits %s %s" % (dtype, model))
    hook = _hook(labels, path, alpha, beta, beam)
    _same(_res(hook, hook.decode_logits(x, sl)), got, "logits %s %s (hook scorer)" % (dtype, model))


def test_config5_equals_hook_scorer_and_reference():
    """BASELINE config 5 as stated: 64 x T=1000 over 29 labels, beam 100, test.arpa, alpha 2.0, beta 1.0"""
    probs, _ = c5_text_probs(48, 1000, seed=71)
    probs = torch.cat([probs, ctc_like_probs(16, 1000, 29, seed=72)], 0)
    dec = _dec(L29, REF_ARPA, 2.0, 1.0, 100)
    got = _res(dec, dec.decode(probs.cuda()))
    hook = _hook(L29, REF_ARPA, 2.0, 1.0, 100)
    _same(_res(hook, hook.decode(probs.cuda())), got, "config 5, hook scorer")
    ref = orc.Reference(L29, model_path=REF_ARPA, alpha=2.0, beta=1.0)
    checked, skipped = compare(ref.decode(probs.numpy(), beam=100), got, None, "config 5, reference build")
    assert checked >= 40, (checked, skipped)
    _same(got, _res(dec, dec.decode(probs)), "config 5, host entry")


def test_character_based_batch_equals_hook_scorer():
    probs = ctc_like_probs(16, 300, len(LCHAR), seed=141)
    dec = _dec(LCHAR, CHAR_LM, 1.3, 0.6, 100)
    assert dec.character_based() and dec.max_order() == 3 and dec.dict_size() == 0
    got = _res(dec, dec.decode(probs.cuda()))
    hook = _hook(LCHAR, CHAR_LM, 1.3, 0.6, 100)
    _same(_res(hook, hook.decode(probs.cuda())), got, "character-based, 16 x 300, beam 100")


@pytest.mark.parametrize("model", ["test", "char"])
def test_streaming_uneven_chunks_equal_offline(model):
    """ctcdec_decode_stream_host in uneven chunks past the arena's first growth (256 frames): at eos the rows equal the
    offline decode, and the committed prefix after every chunk starts every final row"""
    if model == "test":
        labels, path, alpha, beta, beam = L29, REF_ARPA, 2.0, 1.0, 48
        probs, _ = c5_text_probs(3, 700, seed=151)
    else:
        labels, path, alpha, beta, beam = LCHAR, CHAR_LM, 1.3, 0.6, 24
        probs = ctc_like_probs(3, 700, len(LCHAR), seed=152)
    off = _dec(labels, path, alpha, beta, beam)
    want = _res(off, off.decode(probs))
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(labels, model_path=path, alpha=alpha, beta=beta, beam_width=beam,
                                              scorer_provider="device")
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(3)]
    cuts = [0, 50, 187, 188, 488, 700]
    prefixes = []
    for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        eos = b == cuts[-1]
        out = dec.decode(probs[:, a:b], st, [eos] * 3)
        if not eos:
            tok, ts, n_new, committed = dec.committed_prefix(st)
            prefixes.append((tok.numpy(), ts.numpy(), committed.numpy()))
    got = _res(dec, out)
    _same(want, got, "streaming %s" % model)
    for tok, ts, committed in prefixes:
        for b in range(3):
            c = int(committed[b])
            for p in range(int(got["n_results"][b])):
                assert int(got["lens"][b, p]) >= c
                assert np.array_equal(got["tokens"][b, p, :c], tok[b, :c])
                assert np.array_equal(got["timesteps"][b, p, :c], ts[b, :c])


def test_largest_beam_decodes_and_the_next_is_refused():
    probs = text_probs(TEXTS, L29, 60, seed=161)
    dec = _dec(L29, TINY, 1.0, 0.5, 704)
    got = _res(dec, dec.decode(probs.cuda()))
    hook = _hook(L29, TINY, 1.0, 0.5, 704)
    _same(_res(hook, hook.decode(probs.cuda())), got, "beam 704")
    bad = _dec(L29, TINY, 1.0, 0.5, 705)
    with pytest.raises(_native.NativeError, match="error -2: .*with a scorer"):
        bad.decode(probs.cuda())
    _same(got, _res(dec, dec.decode(probs.cuda())), "beam 704 after the refusal")


def test_two_threads_two_device_scorer_decoders_one_device():
    pa = text_probs(TEXTS * 3, L29, 140, seed=131)
    pb = ctc_like_probs(7, 110, len(LCHAR), seed=132)
    da = _dec(L29, TINY, 1.5, 0.8, 32)
    db = _dec(LCHAR, CHAR_LM, 1.3, 0.6, 24)
    want = {"a": _res(da, da.decode(pa)), "b": _res(db, db.decode(pb))}
    errors, done = [], {"a": 0, "b": 0}

    def run(key, dec, probs):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                x = probs.cuda()
                for i in range(3):
                    _same(want[key], _res(dec, dec.decode(x)), "thread %s, round %d" % (key, i))
                    done[key] += 1
        except Exception as e:  # noqa: BLE001 -- reported by the main thread
            errors.append((key, e))
    ts = [threading.Thread(target=run, args=("a", da, pa)), threading.Thread(target=run, args=("b", db, pb))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    assert done == {"a": 3, "b": 3}


def test_refusals_are_followed_by_exact_decodes(tmp_path):
    lib = _native.load()
    probs = text_probs(TEXTS, L29, 100, seed=121)
    dec = _dec(L29, TINY, 1.0, 0.5, 16)
    hook = _hook(L29, TINY, 1.0, 0.5, 16)
    want = _res(hook, hook.decode(probs))
    x = probs.cuda()

    def exact(name):
        _same(want, _res(dec, dec.decode(x)), name)
    exact("before")
    # models the device scorer cannot reproduce exactly
    binary = tmp_path / "model.binary"
    binary.write_bytes(b"mmap lm http://kheafield.com/code\0\0\0\0")
    with pytest.raises(_native.NativeError, match="error -2: .*KenLM binary"):
        _dec(L29, str(binary), 1.0, 0.5, 16)
    exact("after a binary model")
    big = tmp_path / "order7.arpa"
    big.write_text("\\data\\\n" + "".join("ngram %d=1\n" % n for n in range(1, 8)) + "\n")
    with pytest.raises(_native.NativeError, match="order 7 is above 6"):
        _dec(L29, str(big), 1.0, 0.5, 16)
    exact("after an order-7 model")
    # a stream being captured into a CUDA graph
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            with pytest.raises(_native.NativeError, match="error -2: .*CUDA graph"):
                dec.decode(x)
    torch.cuda.current_stream().wait_stream(s)
    del g
    exact("after a capture refusal")
    # a workspace one byte short
    cfg = _native.Config(29, 16, 0, 0, 40, 1.0)
    n = ctypes.c_size_t(0)
    assert lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), dec._scorer.handle, 3, 100, ctypes.byref(n)) == 0
    B, T, K = 3, 100, 16
    out = [torch.empty(B, K, T, dtype=torch.int32, device="cuda") for _ in range(2)]
    sc, ln = torch.empty(B, K, device="cuda"), torch.zeros(B, K, dtype=torch.int32, device="cuda")
    nres, flags = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    rc = lib.ctcdec_decode_batch_lm_device(
        ctypes.byref(cfg), dec._scorer.handle, x.data_ptr(), -1, None, B, T, out[0].data_ptr(), out[1].data_ptr(),
        sc.data_ptr(), ln.data_ptr(), nres.data_ptr(), flags.data_ptr(), None, ws.data_ptr(), n.value - 1,
        torch.cuda.current_stream().cuda_stream)
    assert rc == -4 and b"needed" in lib.ctcdec_last_error()
    exact("after a short workspace")


def test_reset_params_applies_to_the_device_scorer():
    probs = text_probs(TEXTS, L29, 120, seed=171)
    dec = _dec(L29, TINY, 1.0, 0.5, 24)
    hook = _hook(L29, TINY, 1.0, 0.5, 24)
    dec.reset_params(2.5, -0.5)
    hook.reset_params(2.5, -0.5)
    _same(_res(hook, hook.decode(probs.cuda())), _res(dec, dec.decode(probs.cuda())), "after reset_params")
