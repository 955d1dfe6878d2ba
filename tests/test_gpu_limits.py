"""GPU tests at the edges of the launch plan's envelope (the table in tests/test_plan_envelope.py): the largest accepted
beam per vocabulary and the largest accepted vocabulary per beam, through the CUDA-tensor and the host-tensor entry
points, in the latency plan and the throughput plan (B > 264).  The device must equal the CPU emulation of the same
program row for row and flag for flag, and the oracle (or, with a scorer, the reference build) where that is
affordable.  One step past an edge must be refused as unsupported, before anything is launched."""
import os

import numpy as np
import pytest
import torch

from ctcdecode_b200.synth import ctc_like_probs
from oracle import oracle as orc
from tests import emul, tie_inputs
from tests.parity import compare
from tests.test_emulation_edges import EDGES, edge_inputs, kmax, vmax
from tests.test_plan_envelope import MODES, plan_dict

pytestmark = pytest.mark.gpu

L29 = ["_"] + [chr(ord("a") + i) for i in range(26)] + [" ", "'"]
TINY = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "data", "tiny_lm.arpa")


def _decoder(V, beam, labels=None, **kw):
    from ctcdecode_b200 import CTCBeamDecoder
    return CTCBeamDecoder(labels or [str(i) for i in range(V)], beam_width=beam, **kw)


def _rows(dec, out, scores, ts, lens):
    return dict(tokens=out.cpu().numpy(), timesteps=ts.cpu().numpy(), scores=scores.cpu().numpy(),
                lens=lens.cpu().numpy(), n_results=dec.last_n_results.cpu().numpy(),
                ties=dec.last_flags.cpu().numpy())


def _run(probs, seq_lens, beam, on_device, **kw):
    dec = _decoder(probs.shape[2], beam, **kw)
    p = torch.from_numpy(np.ascontiguousarray(probs))
    sl = None if seq_lens is None else torch.from_numpy(np.asarray(seq_lens, np.int32))
    return _rows(dec, *dec.decode(p.cuda() if on_device else p, sl))


def _same_program(want, got, name):
    """Device == emulation: every flag bit, and every row of every utterance, tie-flagged or not."""
    assert np.array_equal(got["ties"], want["ties"]), (name, got["ties"], want["ties"])
    assert not (got["ties"] & 256).any(), name
    a, b = dict(got), dict(want)
    a["ties"] = b["ties"] = np.zeros_like(a["ties"])
    checked, _ = compare(b, a, None, name)
    assert checked == len(a["ties"])
    return checked


@pytest.mark.parametrize("on_device", [True, False], ids=["cuda", "host"])
@pytest.mark.parametrize("V,mode,beam", EDGES, ids=["V%d_%s_beam%d" % e for e in EDGES])
def test_largest_beam_latency_plan(cport, V, mode, beam, on_device):
    """Four utterances (lengths T, 0, 1, T/2 + 3) at Kmax: device == emulation exactly, and == a permitted output of
    the oracle (the same inputs as tests/test_emulation_edges.py)."""
    cut = MODES[mode](V)
    probs, sl = edge_inputs(V, seed=V + beam, T=30 if beam * V < 100000 else 12)   # (as in test_emulation_edges)
    got = _run(probs, sl, beam, on_device, **cut)
    _same_program(emul.decode(probs, sl, beam=beam, **cut), got, "V%d %s beam %d" % (V, mode, beam))
    ref = cport.decode_alternatives(probs, sl, beam=beam, **cut)
    checked, unresolved = compare(ref, got, ref["ties"], "V%d %s beam %d" % (V, mode, beam))
    assert checked + unresolved == 4 and checked >= 2
    print("V %d %s beam %d (%s): 4 == emulation, %d == oracle, %d junk-tie unresolved"
          % (V, mode, beam, "cuda" if on_device else "host", checked, unresolved))


@pytest.mark.parametrize("on_device", [True, False], ids=["cuda", "host"])
@pytest.mark.parametrize("V,mode", [(6, "none"), (29, "top40"), (256, "cp099"), (1024, "none"), (1500, "top40")])
def test_largest_beam_throughput_plan(cport, V, mode, on_device):
    """B = 300 (> 2 x 132: 128-thread CTAs) at the throughput plan's Kmax, T = 10, ragged: every utterance == the
    emulation of the same plan; a seeded sample of 16 against the oracle where the oracle is fast enough."""
    beam = kmax(V, mode, batch="throughput")
    cut = MODES[mode](V)
    B, T = 300, 10
    probs = ctc_like_probs(B, T, V, seed=V).numpy()
    rng = np.random.RandomState(V)
    sl = rng.randint(0, T + 1, size=B).astype(np.int32)
    sl[:3] = [T, 0, 1]
    pl = plan_dict(B, T, V, beam, **cut)
    assert isinstance(pl, dict) and pl["NT"] == 128
    got = _run(probs, sl, beam, on_device, **cut)
    n = _same_program(emul.decode(probs, sl, beam=beam, **cut), got, "throughput V%d %s beam %d" % (V, mode, beam))
    msg = "throughput V %d %s beam %d: %d == emulation" % (V, mode, beam, n)
    if beam * pl["n_max"] < 100000:   # (the oracle takes seconds per frame beyond)
        pick = np.sort(rng.choice(B, 16, replace=False))
        ref = cport.decode_alternatives(probs[pick], sl[pick], beam=beam, **cut)
        sub = {k: v[pick] for k, v in got.items()}
        checked, unresolved = compare(ref, sub, ref["ties"], msg)
        assert np.array_equal(ref["unresolved"], ref["junk_ties"])   # only ties among -FLT_MAX junk prefixes
        # (6 labels at beam 736 over at most 10 frames: every sampled utterance ends in such a junk tie)
        assert checked + unresolved == 16 and (checked >= 8 or V == 6)
        msg += ", sample of 16: %d == oracle, %d junk-tie unresolved" % (checked, unresolved)
    print(msg)


@pytest.mark.parametrize("nt", [128, 256])
def test_device_equals_emulation_on_tie_prone_rows_at_kmax(monkeypatch, nt):
    """Quantised rows (equal scores at the beam cut in many frames) at the largest beams, block size forced on both
    sides: every row and every flag bit identical."""
    monkeypatch.setenv("CTCDEC_NT", str(nt))
    flagged = 0
    for V, mode in ((6, "none"), (29, "top40"), (29, "cp099")):
        beam, cut = kmax(V, mode), MODES[mode](V)
        probs = tie_inputs.quantised_probs(8, 24, V, seed=V + nt)
        got = _run(probs, None, beam, True, **cut)
        want = emul.decode(probs, beam=beam, nt=nt, **cut)
        _same_program(want, got, "tie-prone V%d %s beam %d nt %d" % (V, mode, beam, nt))
        flagged += int(((want["ties"] & 5) != 0).sum())
    assert flagged >= 12   # (the emulation flags all 24 utterances at either block size)
    print("tie-prone rows at Kmax, nt %d: %d tie-flagged utterances equal row for row" % (nt, flagged))


def _check_lsm(lsm, x, seq_lens):
    """The fused log-softmax against a float64 one: 4e-6, or two float32 ulps where those are coarser."""
    want = torch.log_softmax(x.double(), dim=-1).to(lsm.device)
    for b, n in enumerate(seq_lens.tolist()):
        w, g = want[b, :n], lsm[b, :n].double()
        w32 = w.float().abs()
        ulp = (torch.nextafter(w32, torch.full_like(w32, float("inf"))) - w32).double()
        err = (g - w).abs()
        assert bool((err <= torch.clamp(2 * ulp, min=4e-6)).all()), float(err.max())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("beam,mode,V,T", [(32, "top40", 16384, 12), (8, "none", vmax(8, "none"), 3)],
                         ids=["V16384_top40", "largest_unsorted_V"])
def test_decode_logits_at_largest_vocabulary(cport, dtype, beam, mode, V, T):
    """Logits at the vocabulary-sort limit (P = 16384: one warp per prune CTA, 198 KB of keys and staging row) and at
    the largest unsorted vocabulary for beam 8 (a 43 KB staging row, one-frame tiles)."""
    cut = MODES[mode](V)
    x = ctc_like_probs(2, T, V, seed=V + beam, raw_logits=True).to(dtype).cuda()
    seq_lens = torch.tensor([T, 1], dtype=torch.int32)
    dec = _decoder(V, beam, **cut)
    out, scores, ts, lens, lsm = dec.decode_logits(x, seq_lens, return_log_probs=True)
    _check_lsm(lsm, x, seq_lens)
    lsm_cpu = lsm.cpu()
    for b, n in enumerate(seq_lens.tolist()):
        lsm_cpu[b, n:] = 0.0
    want = cport.decode_alternatives(lsm_cpu.numpy(), seq_lens.numpy(), beam=beam, log_input=True, **cut)
    checked, unresolved = compare(want, _rows(dec, out, scores, ts, lens), want["ties"], "logits %s V%d" % (dtype, V))
    assert checked + unresolved == 2 and checked >= 1


def test_pack_results_and_streaming_at_kmax():
    """beam 736 over 29 labels: pack_results of the dense rows; the streaming device entry in chunks of 7 with the
    committed prefix read after every chunk equals the offline decode at eos, and the committed prefix never shrinks
    and starts every final row."""
    import ctcdecode_b200
    beam, B, T = kmax(29, "top40"), 3, 33
    probs = ctc_like_probs(B, T, 29, seed=91)
    dec = ctcdecode_b200.CTCBeamDecoder(L29, beam_width=beam, device_outputs=True)
    out, scores, ts, lens = dec.decode(probs.cuda())
    offsets, ptok, pts = dec.pack_results(out, ts, lens)
    offsets, ptok, pts = offsets.cpu(), ptok.cpu(), pts.cpu()
    off = _rows(dec, out, scores, ts, lens)
    for b in range(B):
        for q in range(beam):
            r = b * beam + q
            n = int(off["lens"][b, q]) if q < int(off["n_results"][b]) else 0
            assert int(offsets[r + 1] - offsets[r]) == n
            assert np.array_equal(ptok[offsets[r]:offsets[r + 1]].numpy(), off["tokens"][b, q, :n])
            assert np.array_equal(pts[offsets[r]:offsets[r + 1]].numpy(), off["timesteps"][b, q, :n])

    sdec = ctcdecode_b200.OnlineCTCBeamDecoder(L29, beam_width=beam)
    st = [ctcdecode_b200.DecoderState(sdec) for _ in range(B)]
    prev = np.zeros(B, np.int64)
    prefix = [np.zeros(0, np.int32)] * B
    for a in range(0, T, 7):
        e = min(T, a + 7)
        res = sdec.decode(probs[:, a:e].cuda(), st, [e == T] * B)
        if e == T:
            break
        tok, _, _, committed = sdec.committed_prefix(st)
        committed = committed.cpu().numpy()
        for b in range(B):
            assert committed[b] >= prev[b] and committed[b] <= e
            t = tok[b, :committed[b]].cpu().numpy()
            assert np.array_equal(t[:prev[b]], prefix[b])
            prefix[b], prev[b] = t, committed[b]
    got = _rows(sdec, *res)
    for b in range(B):
        assert int(got["n_results"][b]) == int(off["n_results"][b])
        for p in range(int(off["n_results"][b])):
            n = int(off["lens"][b, p])
            assert int(got["lens"][b, p]) == n and got["scores"][b, p] == off["scores"][b, p]
            assert np.array_equal(got["tokens"][b, p, :n], off["tokens"][b, p, :n])
            assert np.array_equal(got["timesteps"][b, p, :n], off["timesteps"][b, p, :n])
            assert np.array_equal(got["tokens"][b, p, :prev[b]], prefix[b])


needs_provider = pytest.mark.skipif(not os.path.exists(orc.PROVIDER), reason="scorer provider not built")


@needs_provider
@pytest.mark.parametrize("per_frame", [False, True], ids=["persistent", "per_frame_launch"])
def test_scorer_at_its_largest_beam(monkeypatch, per_frame):
    """The scorer kernel's layout (+ dictionary masks) decides its edge: beam 704 over 29 labels with top 40.  That
    beam decodes like the reference build's Scorer path; beam 705 is refused as unsupported, naming the layout size,
    and a decode right after the refusal is still exact."""
    import ctcdecode_b200
    from ctcdecode_b200._native import NativeError
    if per_frame:
        monkeypatch.setenv("CTCDEC_LM_PER_FRAME", "1")
    beam = kmax(29, "top40", scorer=True)
    probs = ctc_like_probs(3, 20, 29, seed=93)
    ref = orc.Reference(L29, model_path=TINY, alpha=1.5, beta=0.8)
    want = ref.decode(probs.numpy(), beam=beam)

    def run(b):
        dec = ctcdecode_b200.CTCBeamDecoder(L29, model_path=TINY, alpha=1.5, beta=0.8, beam_width=b,
                                            scorer_provider=orc.PROVIDER)
        return _rows(dec, *dec.decode(probs.cuda()))

    checked, skipped = compare(want, run(beam), None, "scorer beam %d" % beam)
    assert checked >= 1
    with pytest.raises(NativeError) as e:
        run(beam + 1)
    assert "error -2" in str(e.value) and "with a scorer" in str(e.value) and "bytes of shared memory" in str(e.value)
    torch.cuda.synchronize()
    compare(want, run(beam), None, "scorer beam %d after a refusal" % beam)
    print("scorer beam %d (%s): %d == reference, %d tie-skipped; beam %d: %s"
          % (beam, "per-frame" if per_frame else "persistent", checked, skipped, beam + 1, e.value))


@needs_provider
def test_scorer_stream_state_refused_at_creation():
    """A streaming state with a scorer past the scorer's edge is refused when it is created, not on its first chunk."""
    import ctcdecode_b200
    from ctcdecode_b200._native import NativeError
    beam = kmax(29, "top40", scorer=True) + 1
    dec = ctcdecode_b200.OnlineCTCBeamDecoder(L29, model_path=TINY, alpha=1.5, beta=0.8, beam_width=beam,
                                              scorer_provider=orc.PROVIDER)
    with pytest.raises(NativeError, match="error -2.*with a scorer"):
        ctcdecode_b200.DecoderState(dec)
    plain = ctcdecode_b200.OnlineCTCBeamDecoder(L29, beam_width=beam)   # the same beam without a scorer fits
    ctcdecode_b200.DecoderState(plain).release()


@pytest.mark.parametrize("on_device", [True, False], ids=["cuda", "host"])
def test_refusals_past_every_edge_launch_nothing(cport, on_device):
    """One step past an edge is CTCDEC_E_UNSUPPORTED with the limit in the message, from both entries, and leaves the
    device as it was: a decode right after is bit-exact."""
    from ctcdecode_b200._native import NativeError
    probs = ctc_like_probs(2, 8, 29, seed=95).numpy()
    for V, K, cut, what in ((29, kmax(29, "top40") + 1, {}, "bytes of shared memory"),
                            (1024, kmax(1024, "none") + 1, dict(cutoff_top_n=1024), "bytes of shared memory"),
                            (vmax(8, "none") + 1, 8, dict(cutoff_top_n=vmax(8, "none") + 1), "bytes of shared memory"),
                            (16385, 8, {}, "vocabulary sort (at most 16384)")):
        x = ctc_like_probs(1, 2, V, seed=V).numpy()
        with pytest.raises(NativeError) as e:
            _run(x, None, K, on_device, **cut)
        assert "error -2" in str(e.value) and what in str(e.value), str(e.value)
        torch.cuda.synchronize()
        ref = cport.decode_alternatives(probs, beam=16)
        compare(ref, _run(probs, None, 16, on_device), ref["ties"], "after refusing V%d beam %d" % (V, K))
