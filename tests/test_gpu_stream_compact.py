"""Compaction of streaming states on the GPU (OnlineCTCBeamDecoder.compact, ctcdec_stream_compact).

Every stream runs beside a twin that is fed the same chunks and never compacted: the committed prefix after every
chunk and the results at eos must be equal bit for bit, through the host entry, the device entry and decode_logits,
with and without device n-gram scorers.  After eos a compaction keeps exactly the trie paths of the returned rows."""
import os

import numpy as np
import pytest
import torch

import ctcdecode_b200
from ctcdecode_b200 import _native
from ctcdecode_b200.synth import ctc_like_probs
from oracle import oracle as orc
from tests.parity import compare
from tests.test_lm import c5_text_probs

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not orc.reference_available(), reason="oracle/_ref not built (needs /root/reference)")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = os.path.join(ROOT, "tests", "data", "tiny_lm.arpa")
REF_ARPA = os.path.join(ROOT, "tests", "golden", "test.arpa")
BUILD_BINARY = os.path.join(ROOT, "oracle", "_ref", "build_binary")
L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]


def _rows(out, dec):
    o, sc, ts, ln = (t.cpu() for t in out)
    return dict(tokens=o.numpy(), timesteps=ts.numpy(), scores=sc.numpy(), lens=ln.numpy(),
                n_results=dec.last_n_results.cpu().numpy(), ties=dec.last_flags.cpu().numpy())


def _same(a, b, name):
    assert np.array_equal(a["n_results"], b["n_results"]) and np.array_equal(a["ties"], b["ties"]), name
    assert np.array_equal(a["lens"], b["lens"]), name
    assert np.array_equal(a["scores"].view(np.int32), b["scores"].view(np.int32)), name
    assert a["tokens"].shape == b["tokens"].shape, name
    for s in range(a["lens"].shape[0]):
        for p in range(int(a["n_results"][s])):
            L = int(a["lens"][s, p])
            assert np.array_equal(a["tokens"][s, p, :L], b["tokens"][s, p, :L]), (name, s, p)
            assert np.array_equal(a["timesteps"][s, p, :L], b["timesteps"][s, p, :L]), (name, s, p)


def _prefixes(r, s):
    """distinct token prefixes (the empty one included) of stream s's returned rows"""
    out = {()}
    for p in range(int(r["n_results"][s])):
        row = tuple(int(x) for x in r["tokens"][s, p, :int(r["lens"][s, p])])
        out.update(row[:i] for i in range(len(row) + 1))
    return len(out)


def _same_committed(dec, a_states, b_states, name):
    """committed depths equal, and each row's new positions (columns past n_new[b] are not written)"""
    ta, sa, na, ca = (x.cpu() for x in dec.committed_prefix(a_states))
    tb, sb, nb, cb = (x.cpu() for x in dec.committed_prefix(b_states))
    assert torch.equal(na, nb) and torch.equal(ca, cb), name
    for r, n in enumerate(na.tolist()):
        assert torch.equal(ta[r, :n], tb[r, :n]) and torch.equal(sa[r, :n], sb[r, :n]), (name, r)


def _twins(decs, model_of, probs, F, every, feed, name):
    """Streams of decoders decs[model_of[s]] and their never-compacted twins, fed chunks of F frames through
    feed(dec, chunk, states, eos) (decs[0] decodes every chunk); compaction after every `every`-th chunk.  Compares the
    committed prefix after every chunk and the rows at eos; returns the eos rows and the compacted states."""
    B, T, _ = probs.shape
    st = [ctcdecode_b200.DecoderState(decs[m]) for m in model_of]
    tw = [ctcdecode_b200.DecoderState(decs[m]) for m in model_of]
    nch = -(-T // F)
    for c in range(nch):
        chunk = probs[:, c * F:(c + 1) * F].contiguous()
        eos = [c == nch - 1] * B
        got = feed(decs[0], chunk, st, eos)
        got = _rows(got, decs[0])
        want = _rows(feed(decs[0], chunk, tw, eos), decs[0])
        if eos[0]:
            _same(want, got, "%s: eos rows" % name)
        if (c + 1) % every == 0 and not eos[0]:
            kept = decs[0].compact(st)
            assert kept.dtype == torch.int64 and kept.shape == (B,) and (kept >= 1).all()
        _same_committed(decs[0], st, tw, "%s: committed prefix after chunk %d" % (name, c))
    return got, st


def _host(dec, chunk, states, eos):
    return dec.decode(chunk.cpu(), states, eos)


def _device(dec, chunk, states, eos):
    return dec.decode(chunk.cuda(), states, eos)


def _logits(dec, chunk, states, eos):
    return dec.decode_logits(chunk.cuda().log().to(torch.float16), states, eos)


@pytest.mark.parametrize("entry", ["host", "device", "device_outputs", "logits"])
@pytest.mark.parametrize("every", [1, 3])
def test_no_scorer_twins(entry, every):
    kw = dict(device_outputs=True, non_blocking=True) if entry == "device_outputs" else {}
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(L29, beam_width=32, **kw)
    probs = ctc_like_probs(5, 300, 29, seed=70 + every)
    feed = dict(host=_host, device=_device, device_outputs=_device, logits=_logits)[entry]
    rows, st = _twins([dec], [0] * 5, probs, 23, every, feed, entry)
    kept = dec.compact(st)  # after eos: the trie paths of the returned rows, nothing else
    assert [int(k) for k in kept] == [_prefixes(rows, s) for s in range(5)]


def _online(model, alpha, beta, beam, device_entry):
    extra = dict(device_outputs=True, non_blocking=True) if device_entry else {}
    return ctcdecode_b200.OnlineCTCBeamDecoder(L29, model_path=model, alpha=alpha, beta=beta, beam_width=beam,
                                               scorer_provider="device", **extra)


@pytest.mark.parametrize("entry", ["host", "device"])
def test_two_device_scorers_in_one_call(entry):
    decs = [_online(REF_ARPA, 1.5, 0.8, 24, entry == "device"), _online(TINY, 2.0, -1.0, 24, entry == "device")]
    probs, _ = c5_text_probs(4, 120, seed=9)
    rows, st = _twins(decs, [0, 1, 1, 0], probs, 17, 2, _device if entry == "device" else _host, entry)
    kept = decs[0].compact(st)
    assert [int(k) for k in kept] == [_prefixes(rows, s) for s in range(4)]


@needs_ref
@pytest.mark.parametrize("entry", ["host", "device"])
def test_two_device_scorers_against_the_reference(entry):
    """compacted after every chunk, states of two device-scorer decoders in one call per chunk against the states of
    two reference decoders in one decode_with_states call per chunk"""
    models = [(REF_ARPA, 1.5, 0.8), (TINY, 2.0, -1.0)]
    beam, F = 16, 30
    decs = [_online(m, a, b, beam, entry == "device") for m, a, b in models]
    refs = [orc.Reference(L29, model_path=m, alpha=a, beta=b) for m, a, b in models]
    probs, _ = c5_text_probs(4, 3 * F, seed=8)
    model_of = [0, 1, 1, 0]
    st = [ctcdecode_b200.DecoderState(decs[m]) for m in model_of]
    rst = [refs[m].state_new(beam) for m in model_of]
    try:
        for c in range(3):
            chunk = probs[:, F * c:F * (c + 1)].contiguous()
            eos = [c == 2] * 4
            out = decs[0].decode(chunk.cuda() if entry == "device" else chunk, st, eos)
            want = refs[0].decode_with_states(chunk.numpy(), rst, eos, beam, max_len=4 * F)
            decs[0].compact(st)
        got = _rows(out, decs[0])
        n = got["tokens"].shape[2]
        for s in range(4):
            g = {k: v[s:s + 1] for k, v in got.items()}
            w = dict(tokens=want["tokens"][s:s + 1, :, :n], timesteps=want["timesteps"][s:s + 1, :, :n],
                     scores=want["scores"][s:s + 1], lens=want["lens"][s:s + 1], n_results=g["n_results"])
            compare(w, g, None, "%s stream %d" % (entry, s))
    finally:
        for r in rst:
            refs[0].state_free(r)


@pytest.mark.skipif(not os.path.exists(BUILD_BINARY), reason="oracle/_ref/build_binary not built")
def test_kenlm_binary_state(tmp_path):
    from tests.test_kenlm_binary import build_binary
    model = build_binary(REF_ARPA, tmp_path, "trie")
    dec = _online(model, 1.0, 1.0, 24, True)
    probs, _ = c5_text_probs(3, 100, seed=10)
    _twins([dec], [0, 0, 0], probs, 13, 2, _device, "kenlm trie")


def test_long_stream():
    """4 streams x 30 000 frames, chunks of 250, beam 100, compaction every 4 chunks: right after each compaction a
    state holds max(1 + beam x 256, kept + beam x 256) nodes of arena and its state block, and decoding grows that as
    the arena rule says (room for kept + beam x frames since, doubling); the twin's arena holds at least
    1 + beam x frames nodes"""
    B, T, F, K = 4, 30000, 250, 100
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(L29, beam_width=K, device_outputs=True, non_blocking=True)
    probs = ctc_like_probs(B, T, 29, seed=77).cuda()
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    tw = [ctcdecode_b200.DecoderState(dec) for _ in range(B)]
    block = 4 * (4 + 12 * K + 6 * 2 * 128)  # state_ints(100) (KP = 128)
    cap = [1 + K * 256] * B
    base, since = [1] * B, 0
    for c in range(T // F):
        since += F
        for s in range(B):
            need = base[s] + K * since
            cap[s] = max(need, 2 * cap[s]) if need > cap[s] else cap[s]
        chunk = probs[:, c * F:(c + 1) * F]
        eos = [c == T // F - 1] * B
        got = _rows(dec.decode(chunk, st, eos), dec)
        want = _rows(dec.decode(chunk, tw, eos), dec)
        if (c + 1) % 4 == 0 and not eos[0]:
            kept = dec.compact(st)
            base, since = [int(k) for k in kept], 0
            cap = [max(1 + K * 256, k + K * 256) for k in base]
        for s in range(B):
            assert st[s].device_bytes() == 32 * cap[s] + block, (c, s)
    _same(want, got, "long stream")
    _same_committed(dec, st, tw, "long stream")
    for s in range(B):
        assert tw[s].device_bytes() >= 32 * (1 + K * T)
        assert st[s].device_bytes() < tw[s].device_bytes()


@needs_ref
def test_hook_scorer_state_is_refused():
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(L29, model_path=TINY, alpha=1.0, beta=1.0, beam_width=8,
                                              scorer_provider=orc.PROVIDER)
    st = [ctcdecode_b200.DecoderState(dec)]
    tw = [ctcdecode_b200.DecoderState(dec)]
    probs = ctc_like_probs(1, 40, 29, seed=3)
    dec.decode(probs[:, :20], st, [False])
    dec.decode(probs[:, :20], tw, [False])
    with pytest.raises(_native.NativeError, match="hook scorer"):
        dec.compact(st)
    _same(_rows(dec.decode(probs[:, 20:], tw, [True]), dec), _rows(dec.decode(probs[:, 20:], st, [True]), dec),
          "after a refusal")


def test_refused_during_graph_capture():
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(L29, beam_width=16, device_outputs=True, non_blocking=True)
    st = [ctcdecode_b200.DecoderState(dec) for _ in range(2)]
    tw = [ctcdecode_b200.DecoderState(dec) for _ in range(2)]
    probs = ctc_like_probs(2, 60, 29, seed=4).cuda()
    dec.decode(probs[:, :30], st, [False, False])
    dec.decode(probs[:, :30], tw, [False, False])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    buf = torch.zeros(1, device="cuda")
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        buf.add_(1)  # (a graph with a node in it)
        with pytest.raises(_native.NativeError, match="CUDA graph"):
            dec.compact(st)
    got = _rows(dec.decode(probs[:, 30:], st, [True, True]), dec)
    _same(_rows(dec.decode(probs[:, 30:], tw, [True, True]), dec), got, "after a refusal")
