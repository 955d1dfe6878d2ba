"""Decoding with the device n-gram scorer without the host (-m gpu): non_blocking=True enqueues the decode and its read-out
rescoring on the stream (ctcdec_decode_batch_lm_device_async, ctcdec_decode_stream_device with ARPA-scorer states).
Every result must equal, bit for bit, the blocking device entry, whose read-out runs on the host."""
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
from tests.test_gpu_ngram_scorer import _logits, _res, _same
from tests.test_lm import c5_text_probs
from tests.test_lm_readout import LCHAR as LCHAR_X, LWORD, adversarial_rows, arpa_scorer, lib_readout, pack

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)"),
]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
CHAR_LM = os.path.join(ROOT, "tests", "data", "char_lm.arpa")
REF_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
LCHAR = ["_"] + list("abcdefghijklmnop") + ["|", "'", "é", " ", "z", "qu"]
TEXTS = ["the cat sat on the mat", "a dog ran fast", "the dog sat on a mat the cat ran"]


def _blocking(labels, model, alpha, beta, beam, **kw):
    return ctcdecode_b200.CTCBeamDecoder(labels, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                         scorer_provider="device", **kw)


def _async(labels, model, alpha, beta, beam, **kw):
    return ctcdecode_b200.CTCBeamDecoder(labels, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                         scorer_provider="device", device_outputs=True, non_blocking=True, **kw)


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", golden_util.names(lm=True) + golden_util.names_char())
def test_fixtures_equal_the_blocking_entry(name):
    probs, seq_lens, kw, gold, alpha, beta = golden_util.load_lm(name)
    labels, model = (LCHAR, CHAR_LM) if name.startswith("lmchar_") else (L29, TINY)
    opts = dict(cutoff_top_n=kw["cutoff_top_n"], cutoff_prob=kw["cutoff_prob"], log_probs_input=kw["log_input"])
    x = torch.from_numpy(probs).cuda()
    sl = None if seq_lens is None else torch.as_tensor(seq_lens).cuda()
    blk = _blocking(labels, model, alpha, beta, kw["beam"], **opts)
    want = _res(blk, blk.decode(x, sl))
    dec = _async(labels, model, alpha, beta, kw["beam"], **opts)
    got = _res(dec, dec.decode(x, sl))
    _same(want, got, name)
    compare(gold, got, None, name + " (fixture)")


@pytest.mark.parametrize("model", ["tiny", "char"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
def test_logits_equal_the_blocking_entry(dtype, model):
    if model == "tiny":
        labels, path, alpha, beta, beam = L29, TINY, 1.5, 0.7, 32
        probs = text_probs(TEXTS * 2, L29, 150, seed=81)
    else:
        labels, path, alpha, beta, beam = LCHAR, CHAR_LM, 1.3, 0.6, 24
        probs = ctc_like_probs(6, 120, len(LCHAR), seed=82)
    x = _logits(probs, dtype, 83)
    sl = torch.tensor([150, 0, 1, 77, 149, 120], dtype=torch.int32).clamp(max=probs.shape[1])
    blk = _blocking(labels, path, alpha, beta, beam)
    *res, lsm_b = blk.decode_logits(x, sl, return_log_probs=True)
    want = _res(blk, res)
    dec = _async(labels, path, alpha, beta, beam)
    *res, lsm = dec.decode_logits(x, sl.cuda(), return_log_probs=True)
    _same(want, _res(dec, res), "logits %s %s" % (dtype, model))
    for b, n in enumerate(sl.tolist()):  # (frames past an utterance's length are not written)
        assert torch.equal(lsm[b, :n].cpu(), lsm_b[b, :n].cpu()), b


def test_config5_equals_blocking_entry_and_reference():
    """config 5 as stated: 64 x T=1000 over 29 labels, beam 100, test.arpa, alpha 2.0, beta 1.0"""
    probs, _ = c5_text_probs(48, 1000, seed=71)
    probs = torch.cat([probs, ctc_like_probs(16, 1000, 29, seed=72)], 0)
    x = probs.cuda()
    blk = _blocking(L29, REF_ARPA, 2.0, 1.0, 100)
    want = _res(blk, blk.decode(x))
    dec = _async(L29, REF_ARPA, 2.0, 1.0, 100)
    got = _res(dec, dec.decode(x))
    _same(want, got, "config 5")
    ref = orc.Reference(L29, model_path=REF_ARPA, alpha=2.0, beta=1.0)
    checked, skipped = compare(ref.decode(probs.numpy(), beam=100), got, None, "config 5, reference build")
    assert checked >= 40, (checked, skipped)


@pytest.mark.parametrize("path,labels", [(REF_ARPA, LWORD), (TINY, LWORD), (CHAR_LM, LCHAR_X)],
                         ids=["test.arpa", "tiny_lm", "char_lm"])
def test_rescore_rows_host_and_device_agree(path, labels):
    tok, lens, nres, scores = pack(adversarial_rows(path, labels, n_random=3000, seed=23), 16, seed=24)
    for alpha, beta in [(2.0, 1.0), (0.7, -1.3)]:
        h = arpa_scorer(path, labels, alpha, beta)
        try:
            host = lib_readout(h, tok, lens, nres, scores, device=-1)
            dev = lib_readout(h, tok, lens, nres, scores, device=torch.cuda.current_device())
        finally:
            _native.load().ctcdec_scorer_destroy(h)
        assert np.array_equal(host.view(np.int32), dev.view(np.int32)), (path, alpha, beta)


def test_graph_capture_replays_on_new_inputs():
    x1 = text_probs(TEXTS * 2, L29, 120, seed=201).cuda()
    x2 = ctc_like_probs(6, 120, 29, seed=202).cuda()
    blk = _blocking(L29, TINY, 1.5, 0.8, 32)
    want1, want2 = _res(blk, blk.decode(x1)), _res(blk, blk.decode(x2))
    dec = _async(L29, TINY, 1.5, 0.8, 32)
    static = x1.clone()
    dec.decode(static)  # outside the capture: tables uploaded, kernel limits raised
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = dec.decode(static)
        nres, flags = dec.last_n_results, dec.last_flags
    for x, want, name in [(x1, want1, "replay 1"), (x2, want2, "replay 2"), (x1, want1, "replay 1 again")]:
        static.copy_(x)
        g.replay()
        torch.cuda.synchronize()
        o, s, ts, ln = out
        got = dict(tokens=o.cpu().numpy(), timesteps=ts.cpu().numpy(), scores=s.cpu().numpy(), lens=ln.cpu().numpy(),
                   n_results=nres.cpu().numpy(), ties=flags.cpu().numpy())
        _same(want, got, name)


def test_capture_with_a_fresh_scorer_is_refused_and_the_capture_stays_valid():
    x = text_probs(TEXTS, L29, 80, seed=211).cuda()
    warm = _async(L29, TINY, 1.0, 0.5, 16)
    want = _res(warm, warm.decode(x))  # (kernels prepared for this shape: only the fresh scorer's tables are missing)
    fresh = _async(L29, TINY, 1.0, 0.5, 16)
    y = torch.arange(16, dtype=torch.float32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        with pytest.raises(_native.NativeError, match="error -2: .*decode once outside the capture first"):
            fresh.decode(x)
        z = y * 2
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(z, y * 2)
    _same(want, _res(fresh, fresh.decode(x)), "fresh scorer after the refused capture")


def test_reset_params_applies_to_the_next_call():
    x = text_probs(TEXTS, L29, 120, seed=221).cuda()
    dec = _async(L29, TINY, 1.0, 0.5, 24)
    before = _res(dec, dec.decode(x))
    dec.reset_params(2.5, -0.5)
    blk = _blocking(L29, TINY, 2.5, -0.5, 24)
    want = _res(blk, blk.decode(x))
    got = _res(dec, dec.decode(x))
    _same(want, got, "after reset_params")
    assert not np.array_equal(before["scores"].view(np.int32), got["scores"].view(np.int32))


def test_the_call_does_not_wait():
    probs = text_probs(TEXTS * 2, L29, 200, seed=231)
    blk = _blocking(L29, TINY, 1.5, 0.8, 32)
    want = _res(blk, blk.decode(probs.cuda()))
    dec = _async(L29, TINY, 1.5, 0.8, 32)
    src = (probs.cuda() * 2.0)
    dec.decode(src * 0.5)  # (first use: tables and limits)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)  # about half a second of GPU clock cycles
        x = src * 0.5                     # the input comes from a kernel queued just before the call
        out = dec.decode(x)
        assert not s.query(), "the decode waited for the stream"
        s.synchronize()
        got = _res(dec, out)
    _same(want, got, "behind a sleep")


def _stream_decode(dec, chunks, n, is_logits, cuts):
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(n)]
    prefixes, out = [], None
    for a, b in zip(cuts[:-1], cuts[1:]):
        eos = b == cuts[-1]
        fn = dec.decode_logits if is_logits else dec.decode
        out = fn(chunks[:, a:b].contiguous(), st, [eos] * n)
        if not eos:
            tok, ts, n_new, committed = dec.committed_prefix(st)
            prefixes.append((tok.cpu().numpy(), ts.cpu().numpy(), committed.cpu().numpy()))
    return _res(dec, out), prefixes


@pytest.mark.parametrize("kind", ["probs", "f16_logits"])
@pytest.mark.parametrize("model", ["test", "char"])
def test_streaming_uneven_chunks_equal_offline(model, kind):
    if model == "test":
        labels, path, alpha, beta, beam = L29, REF_ARPA, 2.0, 1.0, 48
        probs, _ = c5_text_probs(3, 700, seed=151)
    else:
        labels, path, alpha, beta, beam = LCHAR, CHAR_LM, 1.3, 0.6, 24
        probs = ctc_like_probs(3, 700, len(LCHAR), seed=152)
    off = _blocking(labels, path, alpha, beta, beam)
    if kind == "probs":
        x = probs.cuda()
        want = _res(off, off.decode(x))
    else:
        x = _logits(probs, torch.float16, 153)
        want = _res(off, off.decode_logits(x))
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(labels, model_path=path, alpha=alpha, beta=beta, beam_width=beam,
                                              scorer_provider="device", device_outputs=True, non_blocking=True)
    got, prefixes = _stream_decode(dec, x, 3, kind != "probs", [0, 50, 187, 188, 488, 700])
    _same(want, got, "streaming %s %s" % (model, kind))
    for tok, ts, committed in prefixes:
        for b in range(3):
            c = int(committed[b])
            for p in range(int(got["n_results"][b])):
                assert int(got["lens"][b, p]) >= c
                assert np.array_equal(got["tokens"][b, p, :c], tok[b, :c])
                assert np.array_equal(got["timesteps"][b, p, :c], ts[b, :c])


def test_streaming_mixed_eos_leaves_other_streams_untouched():
    probs, _ = c5_text_probs(3, 300, seed=161)
    x = probs.cuda()
    off = _blocking(L29, REF_ARPA, 2.0, 1.0, 32)
    want0 = _res(off, off.decode(x[:1, :200]))
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(L29, model_path=REF_ARPA, alpha=2.0, beta=1.0, beam_width=32,
                                              scorer_provider="device", device_outputs=True, non_blocking=True)
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(3)]
    dec.decode(x[:, :120], st, [False] * 3)
    tok, sc, ts, ln = dec.decode(x[:, 120:200], st, [True, False, False])
    got = _res(dec, (tok, sc, ts, ln))
    assert got["n_results"][1] == 0 and got["n_results"][2] == 0
    assert not got["tokens"][1:].any() and not got["scores"][1:].any() and not got["lens"][1:].any()
    _same(want0, {k: v[:1] for k, v in got.items()}, "stream 0 at eos")
    want = _res(off, off.decode(x[1:, :300]))
    got = _res(dec, dec.decode(x[1:, 200:300], st[1:], [True, True]))
    _same(want, got, "streams 1, 2 at eos")


def test_hook_scorer_states_are_still_refused():
    if not os.path.exists(orc.PROVIDER):
        pytest.skip("scorer provider (make -C oracle provider) not built")
    with pytest.raises(ValueError, match="scorer_provider"):
        ctcdecode_b200.OnlineCTCBeamDecoder(L29, model_path=TINY, alpha=1.0, beta=0.5, beam_width=8,
                                            scorer_provider=orc.PROVIDER, device_outputs=True, non_blocking=True)
    hook = ctcdecode_b200.OnlineCTCBeamDecoder(L29, model_path=TINY, alpha=1.0, beta=0.5, beam_width=8,
                                               scorer_provider=orc.PROVIDER, device_outputs=True)
    hook._non_blocking = True  # (the ABI refusal itself, past the constructor's check)
    st = [ctcdecode_b200.DecoderState(hook)]
    with pytest.raises(_native.NativeError, match="error -2: .*per-frame host handshake"):
        hook.decode(text_probs(TEXTS[:1], L29, 40, seed=171).cuda(), st, [True])


def test_refusals_are_followed_by_exact_decodes():
    lib = _native.load()
    probs = text_probs(TEXTS, L29, 100, seed=121)
    x = probs.cuda()
    blk = _blocking(L29, TINY, 1.0, 0.5, 16)
    want = _res(blk, blk.decode(x))
    dec = _async(L29, TINY, 1.0, 0.5, 16)

    def exact(name):
        _same(want, _res(dec, dec.decode(x)), name)
    exact("before")
    B, T, K = 3, 100, 16
    cfg = _native.Config(29, K, 0, 0, 40, 1.0)
    out = [torch.empty(B, K, T, dtype=torch.int32, device="cuda") for _ in range(2)]
    sc, ln = torch.empty(B, K, device="cuda"), torch.zeros(B, K, dtype=torch.int32, device="cuda")
    nres, flags = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
    n = ctypes.c_size_t(0)
    assert lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), dec._scorer.handle, B, T, ctypes.byref(n)) == 0
    ws = torch.empty(n.value + 1024, dtype=torch.uint8, device="cuda")

    def call(handle, nbytes):
        return lib.ctcdec_decode_batch_lm_device_async(
            ctypes.byref(cfg), handle, x.data_ptr(), -1, None, B, T, out[0].data_ptr(), out[1].data_ptr(),
            sc.data_ptr(), ln.data_ptr(), nres.data_ptr(), flags.data_ptr(), None, ws.data_ptr(), nbytes,
            torch.cuda.current_stream().cuda_stream)
    # a hook scorer
    if os.path.exists(orc.PROVIDER):
        hook = ctcdecode_b200.CTCBeamDecoder(L29, model_path=TINY, alpha=1.0, beta=0.5, beam_width=K,
                                             scorer_provider=orc.PROVIDER)
        assert call(hook._scorer.handle, n.value) == -2
        assert b"ctcdec_scorer_create_arpa" in lib.ctcdec_last_error()
        exact("after a hook scorer")
    # a workspace one byte short
    assert call(dec._scorer.handle, n.value - 1) == -4 and b"needed" in lib.ctcdec_last_error()
    exact("after a short workspace")
    # past the scorer's largest beam
    bad = _async(L29, TINY, 1.0, 0.5, 705)
    with pytest.raises(_native.NativeError, match="error -2: .*with a scorer"):
        bad.decode(x)
    exact("after beam 705")
    # non_blocking without device outputs
    with pytest.raises(ValueError, match="device_outputs"):
        ctcdecode_b200.CTCBeamDecoder(L29, model_path=TINY, alpha=1.0, beta=0.5, beam_width=K,
                                      scorer_provider="device", non_blocking=True)
    exact("after non_blocking without device_outputs")


def test_two_threads_two_streams_match_serial_results():
    pa = text_probs(TEXTS * 3, L29, 140, seed=131)
    pb = ctc_like_probs(7, 110, len(LCHAR), seed=132)
    da = _async(L29, TINY, 1.5, 0.8, 32)
    db = _async(LCHAR, CHAR_LM, 1.3, 0.6, 24)
    want = {"a": _res(da, da.decode(pa.cuda())), "b": _res(db, db.decode(pb.cuda()))}
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
