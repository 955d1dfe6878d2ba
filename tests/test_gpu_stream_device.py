"""Streaming on the device (H100, -m gpu): OnlineCTCBeamDecoder with CUDA chunks (ctcdec_decode_stream_device) against
the host entry point, the offline decoder and the C oracle, and the committed prefix (ctcdec_stream_committed_device)
against the common prefix of the rows an eos read-out returns."""
import ctypes
import os

import numpy as np
import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200 import _native
from ctcdecode_b200.synth import ctc_like_probs, text_probs
from tests.parity import compare

pytestmark = pytest.mark.gpu

L29 = [str(i) for i in range(29)]


def _online(beam, **kw):
    return ctcdecode_b200.OnlineCTCBeamDecoder(L29[:kw.pop("V", 29)], beam_width=beam, **kw)


def _schedule(rng, B, T, sizes):
    """Ragged chunk calls: per call a chunk width from `sizes` and per stream a length in [0, width]; returns a list
    of per-stream length vectors whose sums are T for every stream."""
    pos = np.zeros(B, np.int64)
    calls = []
    while (pos < T).any():
        w = int(rng.choice(sizes))
        ln = np.minimum(rng.randint(0, w + 1, size=B) if w > 0 else np.zeros(B, np.int64), T - pos)
        if rng.rand() < 0.5:
            ln = np.minimum(np.full(B, w), T - pos)
        calls.append(ln.astype(np.int32))
        pos += ln
    return calls


def _chunk(probs, pos, ln):
    """[B, max(ln), V] rows probs[b, pos[b]:pos[b] + ln[b]], padded with the row before (never read)."""
    B, _, V = probs.shape
    w = int(ln.max()) if len(ln) else 0
    out = np.zeros((B, w, V), np.float32)
    for b in range(B):
        out[b, :ln[b]] = probs[b, pos[b]:pos[b] + ln[b]]
    return torch.from_numpy(out)


def _rows(res, scores, ts, lens, nres, flags):
    return dict(tokens=res.cpu().numpy(), timesteps=ts.cpu().numpy(), scores=scores.cpu().numpy(),
                lens=lens.cpu().numpy(), n_results=nres.cpu().numpy(), ties=flags.cpu().numpy())


def _assert_same_rows(a, b, streams, name):
    """Bit-for-bit: n_results, flags, and rows p < n_results (lens, score bits, tokens / timesteps up to len)."""
    for s in streams:
        n = int(a["n_results"][s])
        assert int(b["n_results"][s]) == n, name
        assert int(a["ties"][s]) == int(b["ties"][s]), name
        assert np.array_equal(a["lens"][s, :n], b["lens"][s, :n]), name
        assert np.array_equal(a["scores"][s, :n].view(np.int32), b["scores"][s, :n].view(np.int32)), name
        for p in range(n):
            L = int(a["lens"][s, p])
            assert np.array_equal(a["tokens"][s, p, :L], b["tokens"][s, p, :L]), (name, s, p)
            assert np.array_equal(a["timesteps"][s, p, :L], b["timesteps"][s, p, :L]), (name, s, p)


def test_device_path_equals_host_path(cport):
    B, T, V, K = 16, 1000, 29, 100
    rng = np.random.RandomState(5)
    probs = ctc_like_probs(B, T, V, seed=51).numpy()
    dec = _online(K, device_outputs=True)
    hs = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    ds = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    calls = _schedule(rng, B, T, [0, 1, 100, 100, 37])
    pos = np.zeros(B, np.int64)
    n_eos = 0
    for i, ln in enumerate(calls):
        last = i == len(calls) - 1
        eos = [True] * B if last else list(rng.rand(B) < 0.15)
        chunk = _chunk(probs, pos, ln)
        sl = torch.from_numpy(ln)
        h = dec.decode(chunk, hs, eos, sl)
        hres = _rows(*h, dec.last_n_results, dec.last_flags)
        d = dec.decode(chunk.cuda(), ds, eos, sl)
        assert d[0].is_cuda and dec.last_n_results.is_cuda
        dres = _rows(*d, dec.last_n_results, dec.last_flags)
        pos += ln
        if any(eos):
            assert d[0].shape == (B, K, int(max(pos[b] for b in range(B) if eos[b])))
            _assert_same_rows(hres, dres, [b for b in range(B) if eos[b]], "call %d" % i)
            assert np.array_equal(hres["n_results"], dres["n_results"])
            n_eos += 1
        else:
            assert d[0].shape == (B, 0, 0) and h[0].shape == (B, 0, 0)
    assert n_eos >= 3 and (pos == T).all()
    fr = ctypes.c_int(0)
    _native.check(_native.load().ctcdec_state_frames(ds[0].state, ctypes.byref(fr)))
    assert fr.value == T  # the arenas grew past their initial 256 frames on the way
    ref = cport.decode_alternatives(probs, beam=K)
    compare(ref, dres, ref["ties"], "device streaming, final")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_decode_logits_chunks_equal_offline(dtype):
    B, T, V, K = 4, 300, 29, 32
    logits = ctc_like_probs(B, T, V, seed=52, raw_logits=True).to(dtype).cuda()
    off = ctcdecode_b200.CTCBeamDecoder(L29, beam_width=K, device_outputs=True)
    want = _rows(*off.decode_logits(logits), off.last_n_results, off.last_flags)
    dec = _online(K, device_outputs=True)
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    for a, b in [(0, 0), (0, 50), (50, 51), (51, 177)]:
        r = dec.decode_logits(logits[:, a:b], st, [False] * B)
        assert r[0].shape == (B, 0, 0)
    got = _rows(*dec.decode_logits(logits[:, 177:], st, [True] * B), dec.last_n_results, dec.last_flags)
    want["ties"] = got["ties"] = want["ties"] & 0  # (TIE_VOCAB of earlier chunks is not kept by the stream)
    _assert_same_rows(want, got, range(B), str(dtype))


def test_default_outputs_match_the_host_path():
    B, T, K = 5, 200, 24
    probs = ctc_like_probs(B, T, 29, seed=53)
    sl = torch.tensor([200, 150, 0, 3, 199], dtype=torch.int32)
    dec = _online(K)
    hs = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    ds = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    for a, b, eos in [(0, 60, [False, True, False, False, False]), (60, 60, [False] * 5), (60, 200, [True] * 5)]:
        cl = torch.clamp(sl - a, 0, b - a).int()
        h = dec.decode(probs[:, a:b], hs, eos, cl)
        hf, hn = dec.last_flags, dec.last_n_results
        d = dec.decode(probs[:, a:b].cuda(), ds, eos, cl)
        for x, y in zip(h, d):
            assert not y.is_cuda and x.shape == y.shape and x.dtype == y.dtype
        assert torch.equal(hn, dec.last_n_results) and torch.equal(hf, dec.last_flags)
        assert torch.equal(h[3], d[3])
        for s in range(B):  # (only [s, p, :len] of rows p < n_results is defined)
            n = int(hn[s])
            assert torch.equal(h[1][s, :n].view(torch.int32), d[1][s, :n].view(torch.int32))
            for p in range(n if eos[s] else 0):
                L = int(h[3][s, p])
                assert torch.equal(h[0][s, p, :L], d[0][s, p, :L]) and torch.equal(h[2][s, p, :L], d[2][s, p, :L])


def test_mixed_host_and_device_chunks_equal_offline():
    B, T, K = 3, 400, 32
    probs = ctc_like_probs(B, T, 29, seed=54)
    off = ctcdecode_b200.CTCBeamDecoder(L29, beam_width=K)
    want = _rows(*off.decode(probs), off.last_n_results, off.last_flags)
    dec = _online(K)
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    dec.decode(probs[:, :130], st, [False] * B)             # host
    dec.decode(probs[:, 130:300].cuda(), st, [False] * B)   # device (arena growth on the way)
    got = _rows(*dec.decode(probs[:, 300:], st, [True] * B), dec.last_n_results, dec.last_flags)  # host
    want["ties"] = got["ties"] = want["ties"] & 0
    _assert_same_rows(want, got, range(B), "host, device, host")


def test_device_chunk_does_not_wait_for_the_gpu():
    B, K = 8, 32
    probs = ctc_like_probs(B, 120, 29, seed=55).cuda()
    dec = _online(K, device_outputs=True)
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    dec.decode(probs[:, :40], st, [False] * B)  # (first call: workspace, kernel attributes)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    torch.cuda._sleep(int(2e9))
    dec.decode(probs[:, 40:80], st, [False] * B)  # 80 frames: no arena growth
    busy = not stream.query()
    torch.cuda.synchronize()
    assert busy, "the chunk call waited for the device"


def _lcp(rows, s):
    n = int(rows["n_results"][s])
    L0 = int(rows["lens"][s, 0])
    t0, s0 = rows["tokens"][s, 0, :L0], rows["timesteps"][s, 0, :L0]
    D = L0
    for p in range(1, n):
        L = min(D, int(rows["lens"][s, p]))
        same = (rows["tokens"][s, p, :L] == t0[:L]) & (rows["timesteps"][s, p, :L] == s0[:L])
        D = L if same.all() else int(np.argmin(same))
    return D, t0[:D], s0[:D]


def test_committed_prefix(cport):
    B, T, K = 8, 400, 16
    rng = np.random.RandomState(7)
    probs = ctc_like_probs(B, T, 29, seed=56).numpy()
    dec = _online(K, device_outputs=True)
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    calls = _schedule(rng, B, T, [0, 1, 40, 90])
    pos = np.zeros(B, np.int64)
    prev = torch.zeros(B, dtype=torch.int32, device="cuda")
    acc = [[] for _ in range(B)], [[] for _ in range(B)]
    n_checked = 0
    for i, ln in enumerate(calls):
        dec.decode(_chunk(probs, pos, ln).cuda(), st, [False] * B, torch.from_numpy(ln))
        pos += ln
        tok, ts, n_new, committed = dec.committed_prefix(st, since=prev)
        assert tok.is_cuda and committed.is_cuda
        ftok, fts, fn, fc = dec.committed_prefix(st)
        assert torch.equal(fc, committed) and torch.equal(fn, fc)
        assert (committed >= prev).all(), "the committed prefix shrank"
        # an eos read-out of the same states now: its rows' common prefix is the committed prefix
        now = _rows(*dec.decode(torch.zeros(B, 0, 29, device="cuda"), st, [True] * B), dec.last_n_results,
                    dec.last_flags)
        ref = cport.decode_alternatives(probs[:, :max(int(pos.max()), 1)], pos.astype(np.int32), beam=K, cap=256)
        for s in range(B):
            D = int(committed[s])
            for k, x in ((0, tok), (1, ts)):
                acc[k][s].extend(x[s, :int(n_new[s])].tolist())
            assert acc[0][s] == ftok[s, :D].tolist() and acc[1][s] == fts[s, :D].tolist()
            Dn, nt, nts = _lcp(now, s)
            assert Dn == D and nt.tolist() == acc[0][s] and nts.tolist() == acc[1][s], (i, s)
            if not ref["unresolved"][s]:
                assert any(_lcp(alt, 0)[0] == D and _lcp(alt, 0)[1].tolist() == acc[0][s] and
                           _lcp(alt, 0)[2].tolist() == acc[1][s] for alt in ref["alternatives"][s]), (i, s)
                n_checked += 1
        prev = committed
        # `since` beyond the committed depth reads from 0
        bt, bts, bn, bc = dec.committed_prefix(st, since=committed + 1)
        assert torch.equal(bc, committed) and torch.equal(bn, committed)
        for s in range(B):
            D = int(committed[s])
            assert torch.equal(bt[s, :D], ftok[s, :D]) and torch.equal(bts[s, :D], fts[s, :D])
    final = now
    for s in range(B):
        D = int(prev[s])
        for p in range(int(final["n_results"][s])):
            assert final["tokens"][s, p, :D].tolist() == acc[0][s] and final["timesteps"][s, p, :D].tolist() == acc[1][s]
    assert int(prev.max()) > 0 and n_checked >= B * len(calls) // 2


def test_committed_prefix_of_a_scorer_state():
    from oracle import oracle as orc
    if not os.path.exists(orc.PROVIDER):
        pytest.skip("scorer provider (make -C oracle provider) not built")
    L = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
    texts = ["the cat sat on the mat", "a dog ran fast"]
    probs = text_probs(texts, L, 200, seed=57)
    tiny = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "tiny_lm.arpa")
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(L, model_path=tiny, alpha=1.5, beta=0.7, beam_width=16,
                                              scorer_provider=orc.PROVIDER)
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(2)]
    with pytest.raises(NotImplementedError):
        dec.decode_logits(probs[:, :4].cuda(), st, [False] * 2)
    got = []
    for a, b in [(0, 70), (70, 140)]:
        dec.decode(probs[:, a:b].cuda(), st, [False] * 2)  # CUDA chunk, scorer: the host path
        got.append(dec.committed_prefix(st))
    assert not got[-1][0].is_cuda and int(got[-1][3].max()) > 0
    res, scores, ts, lens = dec.decode(probs[:, 140:], st, [True] * 2)
    for s in range(2):
        D = int(got[-1][3][s])
        for p in range(int(dec.last_n_results[s])):
            assert torch.equal(res[s, p, :D], got[-1][0][s, :D]) and torch.equal(ts[s, p, :D], got[-1][1][s, :D])


def test_state_on_another_device_and_bad_arguments():
    lib = _native.load()
    dec = _online(8, device_outputs=True)
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(2)]
    p = torch.rand(2, 4, 29, device="cuda").softmax(-1)
    st[1].device = 1  # (as if it lived on cuda:1)
    with pytest.raises(ValueError):
        dec.decode(p, st, [False] * 2)
    st[1].device = 0
    other = _online(8, cutoff_top_n=5)
    mixed = [st[0], ctcdecode_b200.DecoderState(other)]
    h = (ctypes.c_void_p * 2)(*[s.state for s in mixed])
    eos = (ctypes.c_uint8 * 2)(0, 0)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    n = torch.zeros(2, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    assert lib.ctcdec_decode_stream_device(p.data_ptr(), -1, None, 2, 4, h, eos, None, None, 0, None, None,
                                           n.data_ptr(), n.data_ptr(), ws.data_ptr(), ws.numel(), stream) == -2
    assert b"same decoder configuration" in lib.ctcdec_last_error()
    h = (ctypes.c_void_p * 2)(*[s.state for s in st])
    assert lib.ctcdec_decode_stream_device(p.data_ptr(), -1, None, 2, 4, h, eos, None, None, 0, None, None,
                                           n.data_ptr(), n.data_ptr(), ws.data_ptr(), 64, stream) == -4
    eos1 = (ctypes.c_uint8 * 2)(1, 0)
    assert lib.ctcdec_decode_stream_device(p.data_ptr(), -1, None, 2, 4, h, eos1, n.data_ptr(), n.data_ptr(), 3,
                                           n.data_ptr(), n.data_ptr(), n.data_ptr(), n.data_ptr(), ws.data_ptr(),
                                           ws.numel(), stream) == -1
    assert b"out_T" in lib.ctcdec_last_error()
    # a scorer state: the device entry refuses it, the committed read-out takes it
    cond = ctypes.CFUNCTYPE(ctypes.c_double, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.c_int)(
        lambda c, l, k: -1.0)
    hooks = _native.ScorerHooks(None, ctypes.cast(cond, ctypes.c_void_p).value, ctypes.cast(cond, ctypes.c_void_p).value)
    labels = (ctypes.c_char_p * 29)(*([b"_"] + [bytes([97 + i]) for i in range(26)] + [b" ", b"'"]))
    words = (ctypes.c_char_p * 2)(b"ab", b"ba")
    sc = ctypes.c_void_p()
    assert lib.ctcdec_scorer_create(ctypes.byref(hooks), 1.0, 0.5, labels, 29, words, 2, 3, 0, ctypes.byref(sc)) == 0
    cfg = _native.Config(29, 8, 0, 0, 40, 1.0)
    lm_state = ctypes.c_void_p()
    assert lib.ctcdec_state_create_lm(ctypes.byref(cfg), sc, 0, ctypes.byref(lm_state)) == 0
    h1 = (ctypes.c_void_p * 1)(lm_state.value)
    assert lib.ctcdec_decode_stream_device(p.data_ptr(), -1, None, 1, 4, h1, eos, None, None, 0, None, None,
                                           n.data_ptr(), n.data_ptr(), ws.data_ptr(), ws.numel(), stream) == -2
    assert b"scorer" in lib.ctcdec_last_error()
    c = torch.full((1,), -5, dtype=torch.int32, device="cuda")
    assert lib.ctcdec_stream_committed_device(h1, 1, None, c.data_ptr(), None, None, 0, stream) == 0
    assert int(c[0]) == 0
    assert lib.ctcdec_state_destroy(lm_state) == 0 and lib.ctcdec_scorer_destroy(sc) == 0
