"""Parity at BASELINE.json's sizes and over random configurations, on the device (-m gpu): the shapes the round-1
review found thinly covered -- BASELINE config 3 (a batch of several waves: the 128-thread / three-CTAs-per-SM plan, at
T = 1000 and beam 100), config 4 at its full batch of 256, random configurations through the CUDA path itself (not only
its CPU emulation), the test knobs that switch the beam kernel's frame structure, and the host entry point's promise
about rows beyond n_results."""
import numpy as np
import pytest
import torch

from ctcdecode_b200.synth import ctc_like_probs, flat_probs
from tests.parity import compare
from tests.test_gpu_parity import _decoder, _run

pytestmark = pytest.mark.gpu


def _slice(dec, out, scores, ts, lens, sl):
    return dict(tokens=out[sl].cpu().numpy(), timesteps=ts[sl].cpu().numpy(), scores=scores[sl].cpu().numpy(),
                lens=lens[sl].cpu().numpy(), n_results=dec.last_n_results[sl].cpu().numpy(),
                ties=dec.last_flags[sl].cpu().numpy())


def test_config3_shape_throughput_plan_exact_sample(cport):
    """BASELINE config 3's per-GPU shape on one GPU: 640 utterances x T=1000 x V=29, beam 100 -- more than 2 x 132
    utterances, so plan.h picks 128-thread CTAs, three per SM, with the small list segments; 16 sampled utterances are
    compared with the oracle bit for bit, all 640 through the size-independent properties."""
    B, T, V, K = 640, 1000, 29, 100
    probs = ctc_like_probs(B, T, V, seed=33)
    dec = _decoder(V, beam=K, device_outputs=True)
    out, scores, ts, lens = dec.decode(probs.cuda())
    assert int((dec.last_flags & 256).sum()) == 0 and bool((dec.last_n_results == K).all())
    assert bool((scores[:, 1:] >= scores[:, :-1]).all()) and bool((lens <= T).all())
    sl = list(range(0, B, 40))
    assert len(sl) == 16
    ref = cport.decode_alternatives(probs[sl].numpy(), beam=K)
    checked, unresolved = compare(ref, _slice(dec, out, scores, ts, lens, sl), ref["ties"], "config3 shape")
    assert checked == 16
    print("config3 shape: %d prune/vocab-tie utterances checked" % int(((ref["ties"] & 5) != 0).sum()))
    # the same utterances decoded alone (latency plan: 256-thread CTAs) give the same bits
    dec2 = _decoder(V, beam=K, device_outputs=True)
    out2, scores2, ts2, lens2 = dec2.decode(probs[sl].cuda())
    assert torch.equal(scores2, scores[sl]) and torch.equal(lens2, lens[sl])
    # prune / vocabulary ties (checked above against every permitted output): their share stays small on this workload
    assert int(((dec.last_flags & 5) != 0).sum()) <= B // 20


def test_config4_full_batch_exact_sample(cport):
    """BASELINE config 4 at its full batch: [256, 2000, 256], beam 200, cutoff_prob 0.99 (sorted / cut vocabulary);
    6 sampled utterances exact against the oracle."""
    B, T, V, K = 256, 2000, 256, 200
    probs = ctc_like_probs(B, T, V, seed=44)
    dec = _decoder(V, beam=K, cutoff_prob=0.99, device_outputs=True)
    out, scores, ts, lens = dec.decode(probs.cuda())
    assert int((dec.last_flags & 256).sum()) == 0
    assert bool((scores[:, 1:] >= scores[:, :-1]).all()) and bool((lens <= T).all())
    sl = [1, 50, 99, 150, 201, 255]
    ref = cport.decode_alternatives(probs[sl].numpy(), beam=K, cutoff_prob=0.99)
    checked, unresolved = compare(ref, _slice(dec, out, scores, ts, lens, sl), ref["ties"], "config4 full batch")
    assert (checked, unresolved) == (6, 0)
    print("config4 full batch: %d prune/vocab-tie utterances checked" % int(((ref["ties"] & 5) != 0).sum()))
    assert np.array_equal(ref["ties"] != 0, (dec.last_flags[sl].cpu().numpy() & 7) != 0)


@pytest.mark.parametrize("knob", [None, ("CTCDEC_NO_FAST", "1"), ("CTCDEC_NO_FAST", "2"), ("CTCDEC_NO_FAST", "4"),
                                  ("CTCDEC_NT", "128"), ("CTCDEC_NT", "192"), ("CTCDEC_NT", "512")],
                         ids=["default", "general_back_half", "no_head_offload", "no_shared_bin_ranking", "nt128", "nt192",
                              "nt512"])
def test_frame_structure_knobs_config2_shape(cport, monkeypatch, knob):
    """The index-order beam kernel runs a frame as two regions (members | grid walk, then a barrier-free commit) and
    falls back to the general back half on rarer frames; the knobs force the general back half in every frame, switch
    off the head hand-over or the ranking of a shared histogram bin, and change the block size (128: every warp owns
    slots AND walks the grid; 192: two grid-walking warps; 512: the run-time-KP kernel).  Same bits in every case,
    index-order and cut-vocabulary kernels alike."""
    if knob:
        monkeypatch.setenv(*knob)
    for probs, kw in ((ctc_like_probs(6, 1000, 29, seed=60).numpy(), dict(beam=100)),
                      (ctc_like_probs(4, 300, 29, seed=61).numpy(), dict(beam=32)),
                      (ctc_like_probs(4, 200, 40, seed=62).numpy(), dict(beam=64, cutoff_top_n=40)),
                      (ctc_like_probs(3, 200, 29, seed=63).numpy(), dict(beam=256)),
                      (ctc_like_probs(2, 300, 256, seed=65).numpy(), dict(beam=200, cutoff_prob=0.99)),   # cut vocabulary
                      (ctc_like_probs(3, 200, 64, seed=66).numpy(), dict(beam=48, cutoff_top_n=12)),
                      (flat_probs(3, 300, 5, seed=64, temp=1.5).numpy(), dict(beam=24))):
        ref = cport.decode_alternatives(probs, **kw)
        got = _run(probs, **kw)
        compare(ref, got, ref["ties"], "%s %s" % (knob, kw))
        assert np.array_equal(ref["ties"] != 0, (got["ties"] & 7) != 0)
        assert not (got["ties"] & 256).any()


def test_random_configurations_on_the_device(cport):
    """hypothesis: random vocabulary / beam / length / pruning mode / input kind / ragged lengths through the CUDA path
    (the seeded random walk of tests/test_emulation.py covers the same program on the CPU)."""
    from hypothesis import HealthCheck, given, settings, strategies as st

    @settings(max_examples=40, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
    @given(V=st.sampled_from([2, 3, 5, 12, 29, 33, 64, 100, 256]), beam=st.sampled_from([1, 2, 8, 31, 32, 33, 100, 128, 200, 300]),
           T=st.integers(1, 120), B=st.integers(1, 5), mode=st.integers(0, 3), kind=st.integers(0, 2),
           seed=st.integers(0, 10000), blank_last=st.booleans(), ragged=st.booleans(), host=st.booleans())
    def run(V, beam, T, B, mode, kind, seed, blank_last, ragged, host):
        rng = np.random.RandomState(seed)
        kw = dict(beam=beam)
        if mode in (1, 3):
            kw["cutoff_top_n"] = int(rng.randint(1, V + 1))
        if mode in (2, 3):
            kw["cutoff_prob"] = float(rng.choice([0.3, 0.9, 0.99, 0.999]))
        blank = V - 1 if blank_last else 0
        kw["blank_id"] = blank
        if kind == 0:
            probs = ctc_like_probs(B, T, V, seed, peak=float(rng.choice([1.0, 3.0, 8.0])), blank_id=blank).numpy()
        elif kind == 1:
            probs = flat_probs(B, T, V, seed, temp=float(rng.choice([0.5, 1.0, 3.0]))).numpy()
        else:
            probs = ctc_like_probs(B, T, V, seed, peak=8.0, blank_id=blank, log=True).numpy()
            kw["log_input"] = True
        sl = rng.randint(0, T + 1, size=B).astype(np.int32) if ragged else None
        ref = cport.decode_alternatives(probs, sl, **kw)
        got = _run(probs, sl, on_device=not host, **kw)
        compare(ref, got, ref["ties"], str(kw))
        assert np.array_equal(ref["unresolved"], ref["junk_ties"]), "only ties among -FLT_MAX junk stay unresolved"
        assert np.array_equal(ref["ties"] != 0, (got["ties"] & 7) != 0)
        assert not (got["ties"] & 256).any()

    run()


def test_host_entry_leaves_rows_beyond_n_results_alone():
    """include/ctcdecode_b200.h: `scores` / `lens` rows p < n_results[b] are written, nothing else (the reference leaves
    its Python-zero-filled out_seq_len at 0 for unused beams, binding.cpp:79-99).  A long batch, then a short one
    through the same cached device buffers: no stale lengths may leak into the rows the second call did not produce."""
    from ctcdecode_b200 import CTCBeamDecoder
    V, K = 6, 64
    dec = CTCBeamDecoder([str(i) for i in range(V)], beam_width=K)
    long_probs = flat_probs(4, 200, V, seed=1, temp=1.0)
    out, scores, ts, lens = dec.decode(long_probs)                   # fills every row of the cached buffers
    assert bool((dec.last_n_results == K).all()) and int(lens.max()) > 3
    short = flat_probs(4, 1, V, seed=2, temp=1.0)                     # one frame: V - 1 + 1 prefixes < beam
    out, scores, ts, lens = dec.decode(short, torch.tensor([1, 1, 0, 1], dtype=torch.int32))
    nres = dec.last_n_results
    assert nres.tolist() == [V, V, 1, V]
    for b in range(4):
        assert bool((lens[b, int(nres[b]):] == 0).all()), lens[b]
        assert bool((lens[b, :int(nres[b])] <= 1).all())


def test_host_entry_pageable_and_page_locked_destinations_agree():
    """ctcdec_decode_batch_host brings the result rows back either by DMA straight into the caller's arrays (page-locked
    memory) or -- pageable memory -- through its own pinned staging rows and a host-side spread: same bits either way,
    and nothing outside [:max_len] of a row is touched."""
    import ctypes
    from ctcdecode_b200 import _native
    lib = _native.load()
    B, T, V, K = 130, 90, 29, 20            # three utterance groups of the host entry point
    probs = ctc_like_probs(B, T, V, seed=77)
    cfg = _native.Config(V, K, 0, 0, 40, 1.0)
    outs = []
    for pinned in (False, True):
        mk = (lambda *s, dt=torch.int32: torch.full(s, -7, dtype=dt).pin_memory()) if pinned else \
             (lambda *s, dt=torch.int32: torch.full(s, -7, dtype=dt))
        tok, ts, sc, ln = mk(B, K, T), mk(B, K, T), mk(B, K, dt=torch.float32), torch.zeros(B, K, dtype=torch.int32)
        nres, fl = torch.zeros(B, dtype=torch.int32), torch.zeros(B, dtype=torch.int32)
        p = probs.pin_memory() if pinned else probs
        _native.check(lib.ctcdec_decode_batch_host(ctypes.byref(cfg), p.data_ptr(), None, B, T, tok.data_ptr(),
                                                   ts.data_ptr(), sc.data_ptr(), ln.data_ptr(), nres.data_ptr(),
                                                   fl.data_ptr(), 0))
        outs.append((tok, ts, sc, ln, nres))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    tok, ts, sc, ln, nres = outs[0]
    assert bool((nres == K).all()) and int(ln.max()) > 5
    assert bool((tok[:, :, int(ln.max()):] == -7).all())   # columns beyond the longest prefix: untouched


@pytest.mark.parametrize("log_input", [False, True], ids=["probs", "log_probs"])
def test_cutoff_prob_exactly_on_a_partial_sum(cport, log_input):
    """The vocabulary cut compares the reference's double log_sum_exp chain (decoder_utils.cpp:26-31) with cutoff_prob.
    The scan kernel decides with a prefix sum and, within 1e-9 of the threshold, replays that chain -- with the glibc
    restatements of double exp / log (glibc_math.cuh), so the decision is the reference's own even when cutoff_prob IS
    a partial sum of the chain, or one ulp to either side of it: every frame of this input sits on that knife edge."""
    import ctypes
    libm = ctypes.CDLL("libm.so.6")
    for f in (libm.exp, libm.log):
        f.restype, f.argtypes = ctypes.c_double, [ctypes.c_double]
    rng = np.random.default_rng(91)
    V, B, T, K, cut = 24, 3, 40, 12, 7
    base = np.sort(rng.dirichlet(np.ones(V) * 0.6).astype(np.float32))[::-1].copy()
    assert len(set(base.tolist())) == V
    vals = np.log(base.astype(np.float64)).astype(np.float32) if log_input else base
    cum = 0.0                                                   # the reference's chain over the sorted row
    for i in range(cut):
        term = float(vals[i]) if log_input else libm.log(float(vals[i]))
        m = max(cum, term)
        cum = libm.log(libm.exp(cum - m) + libm.exp(term - m)) + m
    probs = np.empty((B, T, V), np.float32)
    for b in range(B):
        for t in range(T):
            probs[b, t] = vals[rng.permutation(V)]
    for cp in (cum, float(np.nextafter(cum, 2.0)), float(np.nextafter(cum, 0.0))):
        ref = cport.decode_alternatives(probs, beam=K, cutoff_prob=cp, cutoff_top_n=V, log_input=log_input)
        for on_device in (True, False):
            got = _run(probs, on_device=on_device, beam=K, cutoff_prob=cp, cutoff_top_n=V, log_input=log_input)
            compare(ref, got, ref["ties"], "cutoff_prob %r on the chain's partial sum %d" % (cp, cut))
