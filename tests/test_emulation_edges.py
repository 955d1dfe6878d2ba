"""Host-logic tests (no GPU) at the edges of the launch plan's envelope (tests/test_plan_envelope.py): the CTA
program, emulated on the CPU, against the oracle at the largest accepted beam per vocabulary and the largest accepted
vocabulary per beam.  There the generic-KP kernel runs with up to 736 slots (23 per thread of a 32-lane warp),
list segments are capped by the single-CTA fallback of make_layout, rows longer than 4 KB are staged one frame per
tile, and finalize keeps fewer than 16 checkpoints per round.  Short utterances, ragged lengths including 0 and 1."""
import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, flat_probs
from tests.test_committed_emulation import check_stream
from tests.test_emulation import _check
from tests.test_plan_envelope import BEAMS, KMAX, MODES, VMAX, VOCABS, plan_dict


def kmax(V, mode, scorer=False, batch="latency"):
    return KMAX[(scorer, batch, mode)][VOCABS.index(V)]


def vmax(K, mode, scorer=False, batch="latency"):
    return VMAX[(scorer, batch, mode)][BEAMS.index(K)]


def edge_inputs(V, seed, T=30, B=4):
    probs = ctc_like_probs(B, T, V, seed=seed).numpy()
    return probs, np.array([T, 0, 1, T // 2 + 3][:B], np.int32)


# (V, mode, beam): beam = Kmax, and a few just below it or at a compile-time-KP edge
EDGES = [
    (6, "none", kmax(6, "none")),
    (29, "top40", kmax(29, "top40")),
    (29, "top40", kmax(29, "top40") - 1),           # 735 members in 736 slots: a partly filled last warp
    (29, "cp099", kmax(29, "cp099")),
    (256, "top40", kmax(256, "top40")),
    (256, "cp099", kmax(256, "cp099")),
    (1024, "none", kmax(1024, "none")),
    (1024, "none", 257),                             # first beam of the generic-KP kernel (288 slots)
    (1500, "top40", kmax(1500, "top40")),
]


@pytest.mark.parametrize("V,mode,beam", EDGES, ids=["V%d_%s_beam%d" % e for e in EDGES])
def test_emulation_at_largest_beam(cport, V, mode, beam):
    pl = plan_dict(4, 30, V, beam, **MODES[mode](V))
    assert isinstance(pl, dict) and pl["KP"] >= beam
    # (the oracle takes seconds per frame once beam x labels passes 10^5: shorter utterances there)
    probs, sl = edge_inputs(V, seed=V + beam, T=30 if beam * V < 100000 else 12)
    checked, unresolved = _check(cport, probs, sl, beam=beam, **MODES[mode](V))
    assert checked + unresolved == 4 and checked >= 2   # (lengths 0 and 1 may end in -FLT_MAX junk ties)


VEDGES = [(K, mode, vmax(K, mode)) for K in (1, 32, 100) for mode in ("none", "top40")]


@pytest.mark.parametrize("beam,mode,V", VEDGES, ids=["beam%d_%s_V%d" % e for e in VEDGES])
def test_emulation_at_largest_vocabulary(cport, beam, mode, V):
    pl = plan_dict(3, 20, V, beam, **MODES[mode](V))
    assert isinstance(pl, dict)
    if mode == "none":
        assert pl["F"] == 1          # rows of more than 4 KB: one frame per staged tile
    if beam * V < 100000:
        probs, sl = edge_inputs(V, seed=beam + V, T=20, B=3)
    else:  # (the oracle needs seconds per frame here: 13 s at beam 32 x 10845 labels)
        probs, sl = ctc_like_probs(1, 2, V, seed=beam + V).numpy(), None
    checked, unresolved = _check(cport, probs, sl, beam=beam, **MODES[mode](V))
    assert checked + unresolved == len(probs) and checked >= 1


def test_emulation_largest_beam_in_chunks(cport):
    """Beam 736 over 29 labels through the saved state, 7 frames per chunk."""
    probs, sl = edge_inputs(29, seed=77, T=33)
    _check(cport, probs, sl, chunk=7, beam=kmax(29, "top40"))


def test_committed_program_at_largest_beam(cport):
    """The committed-prefix program after every chunk, and finalize, with 736 members (finalize keeps 11 checkpoints
    per round, committed_cta_run walks 736 members)."""
    probs = ctc_like_probs(1, 16, 29, seed=78).numpy()
    check_stream(cport, probs, None, 8, beam=kmax(29, "top40"))


def test_emulation_random_walk_over_the_envelope(cport):
    """Seeded random walk: vocabularies up to 16384, beams drawn from [1, Kmax(V, mode)], short utterances."""
    rng = np.random.RandomState(4321)
    grid = [V for V in VOCABS if V <= 4096]
    for _ in range(16):
        mode = str(rng.choice(list(MODES)))
        if rng.rand() < 0.25:
            beam = int(rng.choice([1, 8, 32]))
            V = int(rng.randint(2, vmax(beam, mode) + 1))
        else:
            V = int(rng.choice(grid))
            hi = kmax(V, mode)
            beam = int(rng.randint(1, hi + 1)) if rng.rand() < 0.5 else hi
        kw = dict(beam=beam, **MODES[mode](V))
        T, B = int(rng.randint(1, 16)), int(rng.randint(1, 3))
        seed = int(rng.randint(0, 10000))
        probs = ctc_like_probs(B, T, V, seed).numpy() if rng.rand() < 0.7 else flat_probs(B, T, V, seed).numpy()
        sl = rng.randint(0, T + 1, size=B).astype(np.int32) if rng.rand() < 0.5 else None
        _check(cport, probs, sl, chunk=int(rng.choice([0, 0, 5])), **kw)
