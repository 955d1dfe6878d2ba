"""The scorer path with CUDA input (H100, -m gpu): CTCBeamDecoder.decode(cuda_probs) and decode_logits with a language
model go through ctcdec_decode_batch_lm_device, which decodes in place and leaves the results on the GPU.  It must
give exactly what the host entry (ctcdec_decode_batch_lm_host) gives for the same probabilities, and what the
unmodified reference Scorer path gives for the log-softmax the logits scan computed; it must order itself after the
work queued on the caller's stream, refuse what it cannot do and leave the decoder usable afterwards."""
import ctypes
import os
import threading
import time

import numpy as np
import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200 import _native
from ctcdecode_b200.synth import ctc_like_probs, flat_probs, text_probs
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


def _decoder(labels, model, alpha, beta, beam, **kw):
    return ctcdecode_b200.CTCBeamDecoder(labels, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                         scorer_provider=orc.PROVIDER, **kw)


def _res(dec, out):
    o, s, ts, ln = out
    return dict(tokens=o.cpu().numpy(), timesteps=ts.cpu().numpy(), scores=s.cpu().numpy(), lens=ln.cpu().numpy(),
                n_results=dec.last_n_results.cpu().numpy(), ties=dec.last_flags.cpu().numpy())


def _same(want, got, name):
    """bit for bit: n_results, flags, and for every row p < n_results the score bits, the length, and tokens and
    timesteps over [:len]"""
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


def _host_and_device(dec, probs, seq_lens=None):
    """(host entry, device entry) results of the same probabilities"""
    sl = None if seq_lens is None else torch.as_tensor(seq_lens)
    host = _res(dec, dec.decode(probs, sl))
    dev = _res(dec, dec.decode(probs.cuda(), None if sl is None else sl.cuda()))
    return host, dev


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_frame", [False, True], ids=["persistent", "per_frame_launch"])
@pytest.mark.parametrize("name", golden_util.names(lm=True) + golden_util.names_char())
def test_device_entry_equals_host_entry_golden(name, per_frame, monkeypatch):
    if per_frame:
        monkeypatch.setenv("CTCDEC_LM_PER_FRAME", "1")
    probs, seq_lens, kw, gold, alpha, beta = golden_util.load_lm(name)
    labels, model = (LCHAR, CHAR_LM) if name.startswith("lmchar_") else (L29, TINY)
    dec = _decoder(labels, model, alpha, beta, kw["beam"], cutoff_top_n=kw["cutoff_top_n"],
                   cutoff_prob=kw["cutoff_prob"], log_probs_input=kw["log_input"])
    host, dev = _host_and_device(dec, torch.from_numpy(probs), seq_lens)
    _same(host, dev, name)
    compare(gold, dev, None, name + " (device entry vs fixture)")


@pytest.mark.parametrize("cfg", [
    dict(alpha=1.5, beta=0.8, beam=32, T=160, seed=11),
    dict(alpha=0.0, beta=0.0, beam=20, T=100, seed=12),
    dict(alpha=0.5, beta=-0.5, beam=48, T=200, seed=13),
    dict(alpha=2.0, beta=1.0, beam=16, T=120, seed=14, cutoff_prob=0.99),
    dict(alpha=2.0, beta=1.0, beam=16, T=120, seed=15, log_input=True),
    dict(alpha=1.0, beta=2.0, beam=4, T=150, seed=16),
    dict(alpha=1.0, beta=0.5, beam=64, T=100, seed=17, noise=True),
    dict(alpha=1.0, beta=0.5, beam=30, T=80, seed=18, flat=True),
])
def test_device_entry_equals_host_entry_configs(cfg):
    """the configurations test_lm.py checks the emulation on, through both entries, and against the reference"""
    cfg = dict(cfg)
    alpha, beta, T, seed, beam = cfg.pop("alpha"), cfg.pop("beta"), cfg.pop("T"), cfg.pop("seed"), cfg.pop("beam")
    if cfg.pop("noise", False):
        probs = ctc_like_probs(3, T, 29, seed=seed)
    elif cfg.pop("flat", False):
        probs = flat_probs(3, T, 29, seed=seed)
    else:
        probs = text_probs(TEXTS, L29, T, seed=seed)
    log_input = cfg.pop("log_input", False)
    if log_input:
        probs = probs.log()
    dec = _decoder(L29, TINY, alpha, beta, beam, log_probs_input=log_input, **cfg)
    host, dev = _host_and_device(dec, probs)
    _same(host, dev, str(cfg))
    ref = orc.Reference(L29, model_path=TINY, alpha=alpha, beta=beta)
    compare(ref.decode(probs.numpy(), beam=beam, log_input=log_input, num_processes=2, **cfg), dev, None, str(cfg))


def test_device_entry_equals_host_entry_edges():
    """a blank label other than 0, ragged lengths with 0 and 1, one utterance, an empty batch, no frames"""
    labels = L29[1:6] + ["_"] + L29[6:]            # blank at index 5, " " still a label
    probs = ctc_like_probs(5, 90, 29, seed=61, blank_id=5)
    dec = _decoder(labels, TINY, 1.2, 0.4, 24, blank_id=5)
    for sl in (None, np.array([90, 0, 1, 37, 2], np.int32)):
        host, dev = _host_and_device(dec, probs, sl)
        _same(host, dev, "blank 5, seq_lens %s" % sl)
        ref = orc.Reference(labels, model_path=TINY, alpha=1.2, beta=0.4)
        compare(ref.decode(probs.numpy(), sl, beam=24, blank_id=5, num_processes=2), dev, None, "blank 5")
    dec = _decoder(L29, TINY, 1.0, 0.5, 16)
    probs = text_probs(TEXTS[:1], L29, 90, seed=62)
    host, dev = _host_and_device(dec, probs)                                           # B = 1
    _same(host, dev, "B = 1")
    for B, T in ((0, 10), (3, 0)):
        host, dev = _host_and_device(dec, torch.zeros(B, T, 29))
        _same(host, dev, "B %d T %d" % (B, T))
        assert dev["tokens"].shape == (B, 16, T) and dev["n_results"].shape == (B,)


def test_config5_shape_through_cuda_probabilities():
    """BASELINE config 5 as stated: 64 x T=1000 over 29 labels, beam 100, the reference's test.arpa, alpha 2.0,
    beta 1.0, from CUDA probabilities, against the reference's own Scorer path"""
    probs, _ = c5_text_probs(48, 1000, seed=71)
    probs = torch.cat([probs, ctc_like_probs(16, 1000, 29, seed=72)], 0)
    ref = orc.Reference(L29, model_path=REF_ARPA, alpha=2.0, beta=1.0)
    want = ref.decode(probs.numpy(), beam=100)
    dec = _decoder(L29, REF_ARPA, 2.0, 1.0, 100)
    got = _res(dec, dec.decode(probs.cuda()))
    checked, skipped = compare(want, got, None, "config 5 through CUDA probabilities")
    assert checked >= 40, (checked, skipped)


# ---------------------------------------------------------------------------------------------------------------
def _logits(probs, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = probs.clamp_min(1e-20).log() * 1.25 + 0.3 * torch.randn(probs.shape, generator=g)
    return x.to(dtype).cuda()


@pytest.mark.parametrize("model", ["tiny", "char"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
def test_logits_with_a_scorer_match_reference(dtype, model):
    """decode_logits with a scorer: the reference, fed the returned log-softmax with log_probs_input=True, gives the same
    results; so does decode() of that log-softmax on a log-input decoder"""
    if model == "tiny":
        labels, path, alpha, beta, beam = L29, TINY, 1.5, 0.7, 32
        probs = text_probs(TEXTS * 2, L29, 150, seed=81)
    else:
        labels, path, alpha, beta, beam = LCHAR, CHAR_LM, 1.3, 0.6, 24
        probs = ctc_like_probs(6, 120, len(LCHAR), seed=82)
    x = _logits(probs, dtype, 83)
    sl = torch.tensor([150, 0, 1, 77, 149, 120], dtype=torch.int32).clamp(max=probs.shape[1])
    dec = _decoder(labels, path, alpha, beta, beam)
    *res, lsm = dec.decode_logits(x, sl, return_log_probs=True)
    got = _res(dec, res)
    assert lsm.is_cuda and lsm.dtype == torch.float32 and lsm.shape == x.shape
    ref = orc.Reference(labels, model_path=path, alpha=alpha, beta=beta)
    want = ref.decode(lsm.cpu().numpy(), sl.numpy(), beam=beam, log_input=True, num_processes=2)
    compare(want, got, None, "logits %s %s" % (dtype, model))
    ldec = _decoder(labels, path, alpha, beta, beam, log_probs_input=True)
    _same(got, _res(ldec, ldec.decode(lsm.cuda(), sl)), "decode(lsm) on a log-input decoder")
    assert dec.decode_logits(x, sl)[0].shape == got["tokens"].shape    # (without return_log_probs: four tensors)


def test_f16_logits_with_minus_inf_blank():
    """an fp16 -inf blank logit in some frames: the scorer's blank_prob trailer is -inf there"""
    probs = text_probs(TEXTS, L29, 120, seed=91)
    x = _logits(probs, torch.float16, 92)
    x[0, 10:20, 0] = float("-inf")
    x[1, ::7, 0] = float("-inf")
    x[2, 50, :] = 0.0
    x[2, 50, 0] = float("-inf")
    dec = _decoder(L29, TINY, 2.0, 1.0, 32)
    *res, lsm = dec.decode_logits(x, return_log_probs=True)
    got = _res(dec, res)
    assert torch.isinf(lsm[0, 10:20, 0]).all() and torch.isinf(lsm[1, ::7, 0]).all()
    ref = orc.Reference(L29, model_path=TINY, alpha=2.0, beta=1.0)
    compare(ref.decode(lsm.cpu().numpy(), beam=32, log_input=True, num_processes=2), got, None, "fp16 -inf blank")
    ldec = _decoder(L29, TINY, 2.0, 1.0, 32, log_probs_input=True)
    _same(got, _res(ldec, ldec.decode(lsm)), "decode(lsm) with -inf blank")


def test_device_outputs_with_a_scorer():
    probs = text_probs(TEXTS * 2, L29, 130, seed=101)
    sl = torch.tensor([130, 90, 0, 1, 130, 64], dtype=torch.int32)
    dec = _decoder(L29, TINY, 1.5, 0.8, 32)
    want = _res(dec, dec.decode(probs.cuda(), sl))
    ddec = _decoder(L29, TINY, 1.5, 0.8, 32, device_outputs=True)
    out = ddec.decode(probs.cuda(), sl)
    assert all(t.is_cuda for t in out) and ddec.last_n_results.is_cuda and ddec.last_flags.is_cuda
    got = _res(ddec, out)
    _same(want, got, "device_outputs=True")
    offsets, tok, ts = ddec.pack_results(out[0], out[2], out[3])
    offsets, tok, ts = offsets.cpu().numpy(), tok.cpu().numpy(), ts.cpu().numpy()
    K = 32
    for b in range(probs.shape[0]):
        for p in range(K):
            r = b * K + p
            L = int(got["lens"][b, p]) if p < got["n_results"][b] else 0
            assert offsets[r + 1] - offsets[r] == L
            assert np.array_equal(tok[offsets[r]:offsets[r + 1]], got["tokens"][b, p, :L])
            assert np.array_equal(ts[offsets[r]:offsets[r + 1]], got["timesteps"][b, p, :L])
    # decode_logits with device_outputs too
    x = _logits(probs, torch.bfloat16, 102)
    *o2, lsm = ddec.decode_logits(x, sl, return_log_probs=True)
    assert all(t.is_cuda for t in o2)
    _same(_res(dec, dec.decode_logits(x, sl)), _res(ddec, o2), "decode_logits, device_outputs=True")


# ---------------------------------------------------------------------------------------------------------------
def test_caller_stream_orders_the_decode():
    """the logits come from a kernel enqueued on the caller's non-default stream just before the call; then a sleep on
    that stream holds the decode back for longer than the handshake's 8 s no-progress limit"""
    probs = text_probs(TEXTS * 3, L29, 160, seed=111)
    base = _logits(probs, torch.float32, 112)
    dec = _decoder(L29, TINY, 1.5, 0.8, 32)
    want = _res(dec, dec.decode_logits(base))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        x = torch.mul(base, 1.0)   # produced on s, right before the call
        _same(want, _res(dec, dec.decode_logits(x)), "non-default stream")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        torch.cuda._sleep(int(2.2e10))  # ~11 s at the H100's 1.98 GHz boost clock, longer at lower clocks
        e1.record(s)
        y = torch.mul(base, 1.0)
        t0 = time.perf_counter()
        got = _res(dec, dec.decode_logits(y))
        waited = time.perf_counter() - t0
    assert e0.elapsed_time(e1) > 8000.0 and waited > 8.0, (e0.elapsed_time(e1), waited)
    _same(want, got, "decode held back behind a sleep on the caller's stream")


def _raw(dec, lib, cfg, x, ws_bytes=None, scorer=None):
    """one ctcdec_decode_batch_lm_device call on the current stream; returns the code"""
    B, T, V = x.shape
    K = cfg.beam_size
    out = [torch.empty(B, K, T, dtype=torch.int32, device="cuda") for _ in range(2)]
    sc, ln = torch.empty(B, K, device="cuda"), torch.zeros(B, K, dtype=torch.int32, device="cuda")
    nres, flags = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
    n = ctypes.c_size_t(0)
    scorer = scorer or dec._scorer.handle
    if ws_bytes is None:
        assert lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), scorer, B, T, ctypes.byref(n)) == 0
        ws_bytes = n.value
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")
    return lib.ctcdec_decode_batch_lm_device(
        ctypes.byref(cfg), scorer, x.data_ptr(), -1, None, B, T, out[0].data_ptr(), out[1].data_ptr(), sc.data_ptr(),
        ln.data_ptr(), nres.data_ptr(), flags.data_ptr(), None, ws.data_ptr(), ws_bytes,
        torch.cuda.current_stream().cuda_stream)


def test_refusals_leave_the_decoder_usable():
    lib = _native.load()
    probs = text_probs(TEXTS, L29, 100, seed=121)
    dec = _decoder(L29, TINY, 1.0, 0.5, 16)
    want = _res(dec, dec.decode(probs))                     # host entry
    x = probs.cuda()

    def exact(name):
        _same(want, _res(dec, dec.decode(x)), name)
    exact("before")
    # a stream being captured into a CUDA graph: refused before anything is enqueued (the capture stays valid)
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
    # past the scorer's largest beam (704 over 29 labels)
    cfg = _native.Config(29, 705, 0, 0, 40, 1.0)
    assert _raw(dec, lib, cfg, x, ws_bytes=1 << 20) == -2
    msg = lib.ctcdec_last_error().decode()
    assert "with a scorer" in msg and "227 KB" in msg, msg
    exact("after beam 705")
    # a workspace one byte short
    cfg = _native.Config(29, 16, 0, 0, 40, 1.0)
    n = ctypes.c_size_t(0)
    assert lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), dec._scorer.handle, 3, 100, ctypes.byref(n)) == 0
    assert _raw(dec, lib, cfg, x, ws_bytes=n.value - 1) == -4
    assert b"needed" in lib.ctcdec_last_error()
    exact("after a short workspace")
    assert _raw(dec, lib, cfg, x) == 0                      # (the raw call itself works)
    # a scorer built for another number of labels
    other = _decoder(LCHAR, CHAR_LM, 1.0, 0.5, 16)
    assert _raw(dec, lib, cfg, x, ws_bytes=n.value, scorer=other._scorer.handle) == -1
    assert b"23 labels, decoder has 29" in lib.ctcdec_last_error()
    exact("after a label-count mismatch")


def test_two_threads_two_scorer_decoders_one_device():
    """two threads, each with its own scorer decoder and stream, decode concurrently on one device"""
    pa = text_probs(TEXTS * 3, L29, 140, seed=131)
    pb = ctc_like_probs(7, 110, len(LCHAR), seed=132)
    da = _decoder(L29, TINY, 1.5, 0.8, 32)
    db = _decoder(LCHAR, CHAR_LM, 1.3, 0.6, 24)
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
