"""The oracle is pinned before it is trusted: the plain-C restatement (oracle/ctc_oracle.c) must reproduce
(1) the reference's own known answers (reference tests/test_decode.py:13-32,37-91),
(2) the committed outputs of the unmodified reference build (tests/golden, all beams / timesteps / scores),
(3) the reference build's outputs on seeded inputs (tests/golden/reference_build), and the reference build itself on
those inputs whenever oracle/_ref is present."""
import os

import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, flat_probs
from oracle import oracle as orc
from tests import golden_util, tie_inputs
from tests.parity import compare

VOCAB = ["'", " ", "a", "b", "c", "d", "_"]  # reference tests/test_decode.py:13


def _string(tokens, n):
    return "".join(VOCAB[x] for x in tokens[:n])


def test_reference_known_answers(cport):
    probs, _, kw, _ = golden_util.load("ref_kat_beam20")
    r = cport.decode(probs, **kw)
    assert _string(r["tokens"][0, 0], r["lens"][0, 0]) == "acdc"   # test_beam_search_decoder_1
    assert _string(r["tokens"][1, 0], r["lens"][1, 0]) == "b'a"    # test_beam_search_decoder_2 / _batch
    # SURVEY.md Appendix C.3: full golden values of the reference for these inputs
    assert r["scores"][0, 0] == np.float32(6.480283737182617)
    assert list(r["timesteps"][0, 0, :4]) == [0, 1, 4, 5]
    assert list(r["tokens"][1, 3, :4]) == [3, 0, 2, 0] and list(r["timesteps"][1, 3, :4]) == [0, 2, 4, 4]
    lprobs, _, lkw, _ = golden_util.load("ref_kat_beam20_log")      # test_beam_search_decoder_batch_log
    rl = cport.decode(lprobs, **lkw)
    assert _string(rl["tokens"][0, 0], rl["lens"][0, 0]) == "acdc"
    assert _string(rl["tokens"][1, 0], rl["lens"][1, 0]) == "b'a"
    assert np.allclose(rl["scores"], r["scores"], atol=1e-5)


@pytest.mark.parametrize("name", golden_util.names())
def test_cport_matches_reference_golden(cport, name):
    probs, seq_lens, kw, ref = golden_util.load(name)
    got = cport.decode(probs, seq_lens, **kw)
    checked, skipped = compare(ref, got, got["ties"], name)
    assert checked + skipped == probs.shape[0]
    if not name.startswith(("flat", "cp03")):
        assert skipped == 0
    # and every utterance, tie-flagged or not, is one of the outputs the oracle says the reference may produce; only
    # the -FLT_MAX junk ties of cp03 (SURVEY.md quirk Q6) cannot be enumerated
    alts = cport.decode_alternatives(probs, seq_lens, **kw)
    checked, unresolved = compare(alts, ref, None, name + " (alternatives)")
    assert np.array_equal(alts["unresolved"], alts["junk_ties"])
    assert unresolved == (probs.shape[0] if name.startswith("cp03") else 0)


REFERENCE_BUILD = ["T150_V29_beam48", "T90_V40_beam24_top12", "T60_V300_beam40_cp099", "T80_V29_beam30_cp05",
                   "flat_T100_V29_beam50"]
REFERENCE_BUILD_TIES = ["quant_T24_V5_beam3", "quant_T24_V4_beam8_cp09"]


@pytest.mark.parametrize("name", REFERENCE_BUILD, ids=["cfg%d" % i for i in range(5)])
def test_cport_matches_reference_build(cport, name):
    probs, seq_lens, kw, ref = golden_util.load(os.path.join("reference_build", name))
    got = cport.decode(probs, seq_lens, **kw)
    compare(ref, got, got["ties"], name)
    if orc.reference_available():
        live = orc.Reference([str(i) for i in range(probs.shape[2])]).decode(probs, seq_lens, **kw)
        compare(live, got, got["ties"], name + " (live reference build)")


@pytest.mark.parametrize("name", REFERENCE_BUILD + REFERENCE_BUILD_TIES)
def test_enumerator_admits_reference_build_output(cport, name):
    """The committed output of the unmodified reference build is one of the outputs decode_alternatives enumerates,
    on every utterance.  The quant_* fixtures are full of comparator-equal prefixes at the beam cut, and on several of
    them the reference build keeps a different prefix than the oracle's default -- so this pins the enumeration itself.
    T80_V29_beam30_cp05 ties only among -FLT_MAX junk prefixes: unresolved, and nothing else is."""
    probs, seq_lens, kw, ref = golden_util.load(os.path.join("reference_build", name))
    alts = cport.decode_alternatives(probs, seq_lens, **kw)
    checked, unresolved = compare(alts, ref, None, name)
    assert np.array_equal(alts["unresolved"], alts["junk_ties"])
    assert unresolved == (probs.shape[0] if name == "T80_V29_beam30_cp05" else 0)
    if name in REFERENCE_BUILD_TIES:
        assert (alts["ties"] & 1).sum() >= 6
        assert tie_inputs.resolved_by_alternative(alts, ref) >= 2


def _tie_prone_inputs():
    """Seeded inputs on which the beam cut ties: quantised rows, flat rows over few labels, cutoff_prob, blank last."""
    q = tie_inputs.quantised_probs
    return [
        (q(12, 24, 3, 1, (1.0, 2.0)), dict(beam=5)),
        (q(12, 24, 4, 2), dict(beam=8)),
        (q(12, 24, 5, 3), dict(beam=3, blank_id=4)),
        (q(12, 24, 5, 4, (1.0, 2.0, 3.0)), dict(beam=6, blank_id=4, cutoff_prob=0.9)),
        (q(12, 24, 6, 5, (1.0, 2.0, 3.0, 5.0)), dict(beam=10, blank_id=5)),
        (q(12, 24, 6, 6, (1.0, 2.0, 3.0, 5.0)), dict(beam=10, cutoff_top_n=4)),
        (flat_probs(8, 150, 4, seed=7, temp=1.0).numpy(), dict(beam=8, cutoff_prob=0.9, blank_id=3)),
        (flat_probs(8, 150, 6, seed=8, temp=0.5).numpy(), dict(beam=16, blank_id=5)),
    ]


@pytest.mark.skipif(not orc.reference_available(), reason="needs the reference build (make -C oracle ref)")
def test_enumerator_admits_live_reference_build(cport):
    """The same, against the reference build itself on fresh seeded tie-prone inputs."""
    flagged = by_alternative = 0
    for i, (probs, kw) in enumerate(_tie_prone_inputs()):
        alts = cport.decode_alternatives(probs, cap=256, **kw)
        live = orc.Reference([str(v) for v in range(probs.shape[2])]).decode(probs, **kw)
        compare(alts, live, None, "tie-prone input %d %s" % (i, kw))
        assert not alts["junk_ties"].any()
        flagged += int((alts["ties"] & 1).sum() - alts["unresolved"].sum())
        by_alternative += tie_inputs.resolved_by_alternative(alts, live)
    assert flagged >= 30 and by_alternative >= 5


def test_enumerator_tie_groups_larger_than_the_beam(cport):
    """Beam 2 over 3 labels with a top-2 cut: tie groups of m = 3-4 prefixes straddle a cut of K = 2 while the list of
    prefixes is short, so reordering a group must stay inside the oracle's scratch space (it once wrote past it).
    Every alternative is a well-formed decode, and with the reference build present its output is among them."""
    probs = tie_inputs.quantised_probs(8, 24, 3, 0, (1.0, 2.0))
    alts = cport.decode_alternatives(probs, cap=64, beam=2, cutoff_top_n=2)
    assert not alts["unresolved"].any()
    assert sum(len(a) - 1 for a in alts["alternatives"]) >= 10
    for b in range(8):
        for alt in alts["alternatives"][b]:
            assert int(alt["n_results"][0]) == 2
            for p in range(2):
                L = int(alt["lens"][0, p])
                assert ((alt["tokens"][0, p, :L] >= 1) & (alt["tokens"][0, p, :L] < 3)).all()
                assert ((alt["timesteps"][0, p, :L] >= 0) & (alt["timesteps"][0, p, :L] < 24)).all()
    if orc.reference_available():
        live = orc.Reference([str(v) for v in range(3)]).decode(probs, beam=2, cutoff_top_n=2)
        checked, unresolved = compare(alts, live, None, "beam 2, top-2 cut (live reference build)")
        assert (checked, unresolved) == (8, 0)


def test_enumerator_rejects_a_one_ulp_or_one_frame_change(cport):
    """The check can fail: take an utterance whose output is one of several permitted ones (not the default), and
    change one score by one ulp, or one timestep by one frame -- it must then match none of them."""
    probs = tie_inputs.quantised_probs(16, 24, 5, 3)
    alts = cport.decode_alternatives(probs, beam=3, blank_id=4)
    b = next(b for b in range(16) if not alts["unresolved"][b] and len(alts["alternatives"][b]) > 2)
    good = {k: v.copy() for k, v in alts["alternatives"][b][-1].items()}
    ref = {k: (v[b:b + 1] if k not in ("alternatives",) else [v[b]]) for k, v in alts.items()}
    assert compare(ref, good, None, "unchanged") == (1, 0)
    for p in range(int(good["n_results"][0])):
        bad = {k: v.copy() for k, v in good.items()}
        bad["scores"][0, p] = np.nextafter(bad["scores"][0, p], np.float32(np.inf))
        with pytest.raises(AssertionError, match="equals none"):
            compare(ref, bad, None, "one ulp, row %d" % p)
        L = int(good["lens"][0, p])
        if L:
            bad = {k: v.copy() for k, v in good.items()}
            bad["timesteps"][0, p, L - 1] += 1
            with pytest.raises(AssertionError, match="equals none"):
                compare(ref, bad, None, "one frame, row %d" % p)


@pytest.mark.parametrize("name", golden_util.names() + [os.path.join("reference_build", n) for n in REFERENCE_BUILD])
def test_default_choice_is_decode(cport, name):
    """decode_alternatives' first alternative -- every tie choice 0 -- is decode()'s output, bit for bit, and a decode
    with explicit choice-0 vectors is too."""
    probs, seq_lens, kw, _ = golden_util.load(name)
    plain = cport.decode(probs, seq_lens, **kw)
    alts = cport.decode_alternatives(probs, seq_lens, **kw)
    for b in range(probs.shape[0]):
        first = alts["alternatives"][b][0]
        n = len(cport.decode_choices(probs[b], probs.shape[1] if seq_lens is None else seq_lens[b], (), **kw)[1])
        explicit, _ = cport.decode_choices(probs[b], probs.shape[1] if seq_lens is None else seq_lens[b], (0,) * n, **kw)
        for d in (first, explicit):
            for k in ("tokens", "timesteps", "scores", "lens", "n_results", "ties"):
                assert np.array_equal(d[k][0].view(np.int32), plain[k][b].view(np.int32)), (name, b, k)


def test_cport_streaming_equals_offline(cport):
    """DecoderState::next in chunks == one call (reference ctc_beam_search_decoder.cpp:230-243)."""
    probs = ctc_like_probs(1, 97, 29, seed=21).numpy()
    off = cport.decode(probs, beam=20)
    st = cport.state_new(29, 20)
    for a, b in [(0, 10), (10, 11), (11, 60), (60, 97)]:
        cport.state_next(st, probs[0, a:b])
    on = cport.state_decode(st, 20, 97)
    cport.state_free(st)
    n = on["n_results"]
    assert n == off["n_results"][0]
    assert np.array_equal(on["scores"][:n].view(np.int32), off["scores"][0, :n].view(np.int32))
    assert np.array_equal(on["lens"][:n], off["lens"][0, :n])
    for p in range(n):
        L = on["lens"][p]
        assert np.array_equal(on["tokens"][p, :L], off["tokens"][0, p, :L])
        assert np.array_equal(on["timesteps"][p, :L], off["timesteps"][0, p, :L])
