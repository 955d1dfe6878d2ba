"""Host-logic tests (no GPU): the CUDA CTA program (ctcdecode_b200/csrc/beam_program.cuh), compiled as a
single-threaded emulation (tests/native/emulate_cta.cpp), against the oracle -- beam state machine, exact
radix select, tie handling, trie arena / revive / removal cascade, state save + restore between chunks,
finalize.  Bit-exact: tokens, timesteps, lens, n_results and float32 score bits."""
import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, flat_probs
from tests import emul, golden_util, tie_inputs
from tests.parity import compare


def _check(cport, probs, seq_lens=None, nt=0, chunk=0, **kw):
    """Emulation == one of the outputs the reference may produce, on every utterance; only utterances with ties among
    -FLT_MAX junk prefixes may stay unresolved.  Returns (checked, unresolved)."""
    ref = cport.decode_alternatives(probs, seq_lens, **kw)
    got = emul.decode(probs, seq_lens, nt=nt, chunk=chunk, **kw)
    checked, unresolved = compare(ref, got, ref["ties"], str(kw))
    assert np.array_equal(ref["unresolved"], ref["junk_ties"]), "enumeration exceeded its cap on a finite tie"
    # the emulation must flag exactly the utterances the oracle flags
    assert np.array_equal(ref["ties"] != 0, (got["ties"] & 7) != 0)
    assert not (got["ties"] & 256).any()
    return checked, unresolved


@pytest.mark.parametrize("name", golden_util.names())
def test_emulation_matches_reference_golden(name):
    probs, seq_lens, kw, ref = golden_util.load(name)
    got = emul.decode(probs, seq_lens, **kw)
    compare(ref, got, None, name)


@pytest.mark.parametrize("cfg", [
    dict(B=2, T=50, V=6, seed=1, peak=3.0, beam=4),                     # BASELINE config 1
    dict(B=2, T=250, V=29, seed=2, beam=100),                            # config 2 shape, short
    dict(B=2, T=120, V=29, seed=3, beam=20, log=True),
    dict(B=2, T=100, V=29, seed=4, beam=16, cutoff_top_n=10),
    dict(B=2, T=80, V=64, seed=5, beam=16, cutoff_prob=0.99),
    dict(B=2, T=80, V=29, seed=6, beam=16, cutoff_prob=0.5),
    dict(B=2, T=80, V=29, seed=6, beam=16, cutoff_prob=0.3, cutoff_top_n=5),
    dict(B=1, T=150, V=256, seed=7, beam=200, cutoff_prob=0.99),         # config 4 shape, short
    dict(B=2, T=60, V=29, seed=8, beam=300),                             # beam wider than early candidate sets
    dict(B=2, T=60, V=12, seed=9, beam=8, blank_id=11),
    dict(B=2, T=40, V=29, seed=10, beam=10, cutoff_top_n=1),
    dict(B=2, T=40, V=29, seed=10, beam=10, cutoff_top_n=0),
    dict(B=1, T=30, V=1, seed=11, beam=5),
    dict(B=1, T=30, V=2, seed=12, beam=1),
    dict(B=2, T=100, V=29, seed=13, beam=50, flat=True),
    dict(B=2, T=100, V=29, seed=14, beam=7, flat=True, temp=1.0),
    dict(B=1, T=70, V=600, seed=15, beam=12, cutoff_top_n=600),          # wide unsorted vocabulary
    # tiny vocabularies + flat posteriors: hundreds of dead-anchor revivals per utterance (slow path)
    dict(B=4, T=400, V=4, seed=5, beam=16, flat=True, temp=1.0),
    dict(B=4, T=400, V=4, seed=4, beam=16, flat=True, temp=2.0),
    dict(B=4, T=400, V=3, seed=2, beam=8, flat=True, temp=2.0),
    dict(B=4, T=400, V=5, seed=1, beam=16, flat=True, temp=2.0),
])
def test_emulation_matches_oracle(cport, cfg):
    cfg = dict(cfg)
    B, T, V, seed = cfg.pop("B"), cfg.pop("T"), cfg.pop("V"), cfg.pop("seed")
    peak, log = cfg.pop("peak", 8.0), cfg.pop("log", False)
    if cfg.pop("flat", False):
        probs = flat_probs(B, T, V, seed, temp=cfg.pop("temp", 3.0)).numpy()
    elif V == 1:
        probs = np.ones((B, T, 1), np.float32)
    else:
        probs = ctc_like_probs(B, T, V, seed, peak=peak, blank_id=cfg.get("blank_id", 0), log=log).numpy()
    if log:
        cfg["log_input"] = True
    _check(cport, probs, **cfg)


@pytest.mark.parametrize("nt", [32, 64, 128, 160, 192, 256, 512, 1024])
def test_emulation_any_block_size(cport, nt):
    probs = ctc_like_probs(2, 80, 29, seed=20).numpy()
    _check(cport, probs, nt=nt, beam=40)
    _check(cport, ctc_like_probs(1, 300, 29, seed=24).numpy(), nt=nt, beam=100)


def test_emulation_ragged_and_empty(cport):
    probs = ctc_like_probs(6, 60, 29, seed=21).numpy()
    _check(cport, probs, seq_lens=np.array([60, 0, 1, 17, 59, 1000], np.int32), beam=16)
    _check(cport, probs[:, :0], beam=16)


@pytest.mark.parametrize("chunk", [1, 7, 32])
def test_emulation_streaming_state_roundtrip(cport, chunk):
    """Frames fed chunk by chunk through the stored state == one offline pass (device-resident DecoderState)."""
    probs = ctc_like_probs(3, 90, 29, seed=22).numpy()
    _check(cport, probs, seq_lens=np.array([90, 45, 3], np.int32), chunk=chunk, beam=24)
    p2 = ctc_like_probs(1, 64, 100, seed=23).numpy()
    _check(cport, p2, chunk=chunk, beam=12, cutoff_top_n=15)


@pytest.mark.parametrize("cfg", [
    dict(V=3, beam=5, temp=2.0),
    dict(V=4, beam=8, temp=1.0),
    dict(V=5, beam=10, temp=1.0, blank_id=4, cutoff_prob=0.9),
    dict(V=6, beam=16, temp=0.5, blank_id=5),
    dict(V=6, beam=12, temp=1.0, cutoff_top_n=4),
])
def test_emulation_flat_small_vocabulary_ties(cport, cfg):
    """Flat rows over 3-6 labels: tie-flagged utterances are compared against every output the reference may
    produce, not skipped."""
    cfg = dict(cfg)
    V, temp = cfg.pop("V"), cfg.pop("temp")
    probs = flat_probs(8, 150, V, seed=V, temp=temp).numpy()
    checked, unresolved = _check(cport, probs, **cfg)
    assert checked + unresolved == 8


@pytest.mark.parametrize("cfg", [
    dict(V=3, beam=5, levels=(1.0, 2.0)),
    dict(V=4, beam=8),
    dict(V=5, beam=3, blank_id=4),
    dict(V=5, beam=6, blank_id=4, cutoff_prob=0.9, levels=(1.0, 2.0, 3.0)),
    dict(V=6, beam=10, levels=(1.0, 2.0, 3.0, 5.0)),
    dict(V=6, beam=6, cutoff_top_n=4, levels=(1.0, 2.0, 3.0, 5.0, 7.0)),
    dict(V=6, beam=10, log_input=True, levels=(1.0, 2.0, 3.0, 5.0)),
], ids=["V3", "V4", "V5_beam3", "V5_cp", "V6", "V6_top4", "V6_log"])
@pytest.mark.parametrize("nt", [0, 128])
def test_emulation_quantised_rows_prune_ties(cport, cfg, nt):
    """Probabilities quantised to a few values: equal scores at the beam cut in many frames (TIE_PRUNE).  Every
    utterance must equal one of the outputs the reference may produce.  A few utterances chain so many tie frames that
    their choice vectors exceed the enumeration cap; they count as unresolved and are bounded here."""
    cfg = dict(cfg)
    V, levels = cfg.pop("V"), cfg.pop("levels", (1.0, 2.0, 4.0))
    probs = tie_inputs.quantised_probs(16, 24, V, seed=V + 10 * cfg["beam"], levels=levels)
    if cfg.get("log_input"):
        probs = np.log(probs)
    ref = cport.decode_alternatives(probs, cap=256, **cfg)
    assert (ref["ties"] & 1).sum() >= 6                    # the input does what it is for
    got = emul.decode(probs, nt=nt, **cfg)
    checked, unresolved = compare(ref, got, ref["ties"], str(cfg))
    assert checked + unresolved == 16 and checked >= 13
    assert np.array_equal(ref["ties"] != 0, (got["ties"] & 7) != 0)


def test_emulation_quantised_rows_need_alternatives(cport):
    """The quantised inputs above are not vacuous: on them the CTA program keeps a different (equally ranked) prefix
    than the oracle's default resolution in some utterances, which the old skip-and-count rule never looked at."""
    n = 0
    for V, beam, blank in ((4, 8, 0), (5, 3, 4), (6, 10, 0)):
        probs = tie_inputs.quantised_probs(16, 24, V, seed=V + 10 * beam)
        ref = cport.decode_alternatives(probs, cap=256, beam=beam, blank_id=blank)
        got = emul.decode(probs, beam=beam, blank_id=blank)
        compare(ref, got, ref["ties"], "quantised V%d" % V)
        n += tie_inputs.resolved_by_alternative(ref, got)
    assert n > 0


def test_emulation_config4_row_with_a_finite_prune_tie(cport):
    """A config-4 utterance (T = 2000, V = 256, beam 200, cutoff_prob 0.99) with one finite-score tie at the beam cut
    (frame 1632: two prefixes, one kept).  The oracle decodes it twice; the CTA program must equal one of the two."""
    probs = ctc_like_probs(2, 2000, 256, seed=0).numpy()[1:2]
    ref = cport.decode_alternatives(probs, beam=200, cutoff_prob=0.99)
    assert ref["ties"][0] & 1 and not ref["unresolved"][0]
    got = emul.decode(probs, beam=200, cutoff_prob=0.99)
    assert compare(ref, got, ref["ties"], "config 4, utterance 1") == (1, 0)


@pytest.mark.parametrize("path", list(tie_inputs.PRUNE_PATHS))
@pytest.mark.parametrize("kind", tie_inputs.DEGENERATE)
def test_emulation_degenerate_values(cport, kind, path):
    """Exact zeros, subnormal probabilities, probabilities above 1, one-hot blank frames, -inf / -FLT_MAX / -1e30 /
    positive log-probabilities and blank at -inf for whole stretches, through every vocabulary-cut configuration.
    Unresolved utterances (n_results only) occur in three cells: -FLT_MAX junk ties with cutoff_prob (above_one: 1 of
    6, log_extremes: 3 of 6), and, in log_extremes with the top-40 cut of 256 labels, 2 of 6 whose finite ties chain
    past the enumeration cap (-1e30 absorbs any score it is added to).  Every cell checks at least 3 of its 6
    utterances exactly, and only log_extremes may leave a finite tie unresolved."""
    V, kw = tie_inputs.PRUNE_PATHS[path]
    probs, log_input = tie_inputs.degenerate_probs(kind, 6, 40, V, seed=V)
    ref = cport.decode_alternatives(probs, cap=256, log_input=log_input, **kw)
    got = emul.decode(probs, log_input=log_input, **kw)
    checked, unresolved = compare(ref, got, ref["ties"], "%s %s" % (kind, path))
    assert checked + unresolved == 6 and checked >= 3
    assert (ref["unresolved"] & ~ref["junk_ties"]).sum() == 0 or kind == "log_extremes"
    assert np.array_equal(ref["ties"] != 0, (got["ties"] & 7) != 0)
    assert not (got["ties"] & 256).any()


def test_emulation_uniform_input_massive_ties(cport):
    """All-equal probabilities: every candidate ties.  Results are reference-unspecified (flagged), but the
    program must terminate, keep exactly beam_size prefixes and agree with the oracle on the flag."""
    probs = np.full((1, 12, 5), 0.2, np.float32)
    ref = cport.decode(probs, beam=6)
    got = emul.decode(probs, beam=6)
    assert got["n_results"][0] == ref["n_results"][0] == 6
    assert (got["ties"][0] & 3) != 0 and ref["ties"][0] != 0
    # multiset of scores is still determined
    assert np.array_equal(np.sort(got["scores"][0]), np.sort(ref["scores"][0]))


def test_emulation_grid_fallback_path(cport, monkeypatch):
    """The candidate-list fast path and the grid-walking fallback (taken when a warp's list segment overflows)
    must agree with the oracle -- force the fallback on every frame."""
    monkeypatch.setenv("CTC_EMU_FORCE_FALLBACK", "1")
    _check(cport, ctc_like_probs(2, 150, 29, seed=40).numpy(), beam=60)
    _check(cport, ctc_like_probs(1, 100, 256, seed=41).numpy(), beam=100, cutoff_prob=0.99)
    _check(cport, flat_probs(2, 200, 4, seed=5, temp=1.0).numpy(), beam=16)
    _check(cport, np.full((1, 12, 5), 0.2, np.float32)[:, :0], beam=6)


def test_emulation_segment_overflow_takes_fallback(cport):
    """beam 512 x 40 kept characters: a warp's list segment (capped at 64 KB / warps) cannot hold all candidates of
    its 32 members while the beam is filling up, so early frames overflow into the fallback and later frames use
    the list."""
    probs = ctc_like_probs(1, 12, 64, seed=42).numpy()
    _check(cport, probs, beam=512)


@pytest.mark.parametrize("seg", [8, 40, 150])
def test_emulation_list_overflow_rewalk(cport, monkeypatch, seg):
    """A list segment that overflows makes the frame walk the grid once more with lo32 raised to the lower edge of
    the K-th key's histogram bin (beam_program.cuh, region G); if that overflows too, the grid-walking fallback takes
    over.  Tiny segments force both on ordinary inputs: results must not change."""
    monkeypatch.setenv("CTC_EMU_SEG", str(seg))
    monkeypatch.setenv("CTC_EMU_HEUR_BIAS", "0.7")  # and let the checked bound fail now and then on top of it
    _check(cport, ctc_like_probs(2, 150, 29, seed=50).numpy(), beam=60)
    _check(cport, ctc_like_probs(1, 100, 256, seed=51).numpy(), beam=100, cutoff_prob=0.99)
    _check(cport, ctc_like_probs(2, 80, 64, seed=52).numpy(), beam=32, cutoff_top_n=12)
    _check(cport, flat_probs(2, 200, 4, seed=5, temp=1.0).numpy(), beam=16)


@pytest.mark.parametrize("bias", ["0.5", "3.0", "40.0"])
def test_emulation_checked_bound_failure_is_redone(cport, monkeypatch, bias):
    """Kernels for a per-frame vocabulary cut start the grid walk from a heuristic lower bound of the K-th key
    (lowest beam score + largest non-blank log-prob) that is CHECKED against the histogram total; a bound that cuts
    too deep (forced here by a bias) makes the frame walk again with the proven bound.  Results must not change."""
    monkeypatch.setenv("CTC_EMU_HEUR_BIAS", bias)
    _check(cport, ctc_like_probs(1, 100, 256, seed=51).numpy(), beam=100, cutoff_prob=0.99)
    _check(cport, ctc_like_probs(2, 80, 64, seed=52).numpy(), beam=32, cutoff_top_n=12)
    _check(cport, flat_probs(2, 120, 12, seed=6, temp=1.0).numpy(), beam=16, cutoff_top_n=5)
    _check(cport, ctc_like_probs(2, 150, 29, seed=53).numpy(), beam=60)      # index-order kernel: grid-walking select
    _check(cport, flat_probs(2, 150, 6, seed=7, temp=1.5).numpy(), beam=24)


def test_plan_shapes():
    """plan.h: block size / shared-memory budget by batch size (latency vs throughput shape), slot count rounded to
    the sizes the beam kernel is specialised for, and every layout inside the 227 KB an SM offers."""
    c2 = emul.plan(256, 1000, 29, 100)
    assert (c2["NT"], c2["KP"], c2["budget_kb"], c2["sorted"]) == (256, 128, 111, 0)
    assert 2 * (c2["smem"] + 1024) <= 227 * 1024            # two CTAs per SM
    c3 = emul.plan(2048, 1000, 29, 100)
    assert (c3["NT"], c3["KP"], c3["budget_kb"]) == (128, 128, 74)
    assert 3 * (c3["smem"] + 1024) <= 227 * 1024            # three CTAs per SM
    c4 = emul.plan(256, 2000, 256, 200, cutoff_prob=0.99)
    assert (c4["NT"], c4["KP"], c4["sorted"], c4["NP"]) == (256, 256, 1, 48)
    assert 2 * (c4["smem"] + 1024) <= 227 * 1024
    assert emul.plan(1, 50, 6, 4)["KP"] == 32 and emul.plan(1, 50, 6, 4)["NT"] == 128
    assert [emul.plan(4, 10, 29, k)["KP"] for k in (32, 33, 64, 65, 128, 129, 256, 257, 300)] == \
        [32, 64, 64, 128, 128, 256, 256, 288, 320]
    for k in (1, 16, 100, 256, 512, 1024, 2048):
        for v in (2, 29, 256, 5000):
            pl = emul.plan(8, 20, v, k)
            assert isinstance(pl, int) or pl["smem"] <= 227 * 1024, (k, v, pl)
            if not isinstance(pl, int):
                assert pl["seg"] >= 32
    assert isinstance(emul.plan(8, 20, 29, 5000), int)      # beam size out of range -> an error code, not a layout


@pytest.mark.parametrize("knob", [None, ("CTC_EMU_SEG", "16"), ("CTC_EMU_HEUR_BIAS", "1.5"), ("CTC_EMU_FORCE_FALLBACK", "1")])
def test_emulation_random_configs(cport, monkeypatch, knob):
    """Seeded random walk over vocabulary / beam / length / pruning mode / input kind / ragged lengths / streaming
    chunk size, with the test knobs that force the rare select paths: the CTA program must agree with the oracle."""
    if knob:
        monkeypatch.setenv(*knob)
    rng = np.random.RandomState(1234 + (0 if knob is None else len(knob[0])))
    for _ in range(60):
        V = int(rng.choice([2, 3, 5, 8, 12, 29, 33, 64, 100, 256]))
        beam = int(rng.choice([1, 2, 4, 8, 16, 31, 32, 33, 60, 100, 128, 200]))
        T, B = int(rng.randint(1, 60)), int(rng.randint(1, 4))
        kw = dict(beam=beam)
        mode = rng.randint(0, 4)
        if mode in (1, 3):
            kw["cutoff_top_n"] = int(rng.randint(1, V + 1))
        if mode in (2, 3):
            kw["cutoff_prob"] = float(rng.choice([0.3, 0.9, 0.99, 0.999]))
        blank = int(rng.choice([0, V - 1]))
        kw["blank_id"] = blank
        kind, seed = rng.randint(0, 3), int(rng.randint(0, 10000))
        if kind == 0:
            probs = ctc_like_probs(B, T, V, seed, peak=float(rng.choice([1.0, 3.0, 8.0])), blank_id=blank).numpy()
        elif kind == 1:
            probs = flat_probs(B, T, V, seed, temp=float(rng.choice([0.5, 1.0, 3.0]))).numpy()
        else:
            probs = ctc_like_probs(B, T, V, seed, peak=8.0, blank_id=blank, log=True).numpy()
            kw["log_input"] = True
        sl = rng.randint(0, T + 1, size=B).astype(np.int32) if rng.rand() < 0.5 else None
        chunk = int(rng.choice([0, 0, 1, 7, 16]))
        _check(cport, probs, sl, chunk=chunk, **kw)


@pytest.mark.parametrize("knob", ["1", "2", "4"], ids=["general_back_half", "no_head_offload", "no_shared_bin_ranking"])
@pytest.mark.parametrize("order", ["0", "7"])
def test_emulation_frame_structure_knobs(cport, monkeypatch, knob, order):
    """CTC_EMU_NO_FAST switches parts of the two-region frame off (general back half everywhere / every warp computes
    the head / no ranking of a shared histogram bin); CTC_EMU_ORDER runs the emulated threads in reversed order."""
    monkeypatch.setenv("CTC_EMU_NO_FAST", knob)
    monkeypatch.setenv("CTC_EMU_ORDER", order)
    _check(cport, ctc_like_probs(2, 300, 29, seed=70).numpy(), beam=100)
    _check(cport, ctc_like_probs(1, 150, 256, seed=71).numpy(), beam=200, cutoff_prob=0.99)
    _check(cport, ctc_like_probs(2, 120, 64, seed=72).numpy(), beam=32, cutoff_top_n=12, nt=192)
    _check(cport, flat_probs(2, 200, 5, seed=73, temp=1.5).numpy(), beam=24)
