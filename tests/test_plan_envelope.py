"""The shapes the launch plan accepts (plan.h, no GPU): the largest beam per vocabulary and the largest vocabulary per
beam, for every pruning mode, both batch plans and with and without a scorer, committed below as data.  Every
accepted shape must have a beam-kernel layout whose regions fit the 227 KB of shared memory an H100 CTA can opt into,
and so must the prune, finalize and committed-prefix kernels; one step past an edge must be refused as unsupported,
with a message that names the limit.  A layout change that moves an edge fails here and shows up in review."""
import ctypes
import os
import re
import subprocess

import pytest

SMEM_CTA = 227 * 1024      # cudaDevAttrMaxSharedMemoryPerBlockOptin on the H100
CTCDEC_E_UNSUPPORTED = -2

# pruning modes: nothing cut (the vocabulary is used unsorted), the default top-40 cut, cutoff_prob 0.99 (with top 40)
MODES = {
    "none": lambda V: dict(cutoff_top_n=V),
    "top40": lambda V: dict(cutoff_top_n=40),
    "cp099": lambda V: dict(cutoff_prob=0.99),
}
# batch plans: the latency plan (one wave, B <= 264) and the throughput plan (B > 264)
BATCHES = {"latency": 8, "throughput": 300}
VOCABS = (2, 6, 29, 64, 100, 256, 600, 1024, 1500, 4096, 16384)
BEAMS = (1, 8, 32, 100, 200)

# largest accepted beam, per (scorer, batch plan, mode), for VOCABS (0: no beam fits)
KMAX = {
    (False, "latency", "none"): (736, 736, 736, 672, 640, 544, 416, 320, 128, 64, 0),
    (False, "latency", "top40"): (736, 736, 736, 672, 640, 576, 448, 352, 288, 128, 32),
    (False, "latency", "cp099"): (736, 736, 704, 672, 640, 576, 448, 352, 288, 128, 32),
    (False, "throughput", "none"): (736, 736, 736, 672, 640, 544, 416, 320, 128, 64, 0),
    (False, "throughput", "top40"): (736, 736, 736, 672, 640, 576, 448, 384, 288, 128, 32),
    (False, "throughput", "cp099"): (736, 736, 704, 672, 640, 576, 448, 384, 288, 128, 32),
    (True, "latency", "none"): (736, 736, 704, 640, 608, 512, 352, 256, 128, 64, 0),
    (True, "latency", "top40"): (736, 736, 704, 672, 640, 608, 544, 480, 416, 128, 32),
    (True, "latency", "cp099"): (736, 704, 704, 672, 640, 608, 544, 480, 416, 128, 32),
    (True, "throughput", "none"): (736, 736, 704, 640, 608, 512, 352, 256, 128, 64, 0),
    (True, "throughput", "top40"): (736, 736, 704, 672, 640, 608, 544, 480, 416, 128, 32),
    (True, "throughput", "cp099"): (736, 736, 704, 672, 640, 608, 544, 480, 416, 128, 32),
}
# largest accepted vocabulary, per (scorer, batch plan, mode), for BEAMS; 16384 is the vocabulary-sort limit
VMAX = {
    (False, "latency", "none"): (10845, 10845, 10845, 3389, 1469),
    (False, "latency", "top40"): (16384, 16384, 16384, 4896, 2048),
    (False, "latency", "cp099"): (16384, 16384, 16384, 4896, 2048),
    (False, "throughput", "none"): (10909, 10909, 10909, 3389, 1469),
    (False, "throughput", "top40"): (16384, 16384, 16384, 4928, 2048),
    (False, "throughput", "cp099"): (16384, 16384, 16384, 4928, 2048),
    (True, "latency", "none"): (9053, 9053, 9053, 2621, 1117),
    (True, "latency", "top40"): (16384, 16384, 16384, 8736, 3744),
    (True, "latency", "cp099"): (16384, 16384, 16384, 8736, 3744),
    (True, "throughput", "none"): (9085, 9085, 9085, 2637, 1117),
    (True, "throughput", "top40"): (16384, 16384, 16384, 8792, 3776),
    (True, "throughput", "cp099"): (16384, 16384, 16384, 8792, 3776),
}
CELLS = sorted(KMAX, key=str)


def _ids(cell):
    return "%s-%s-%s" % ("scorer" if cell[0] else "plain", cell[1], cell[2])


_PLAN_KEYS = ("NT", "KP", "budget_kb", "seg", "smem", "F", "NP", "sorted",
              "evcnt", "mask", "mask2", "rmask", "dmask", "rank", "tile_lp", "tile_idx", "clk", "cli",
              "W", "WC", "NW", "P", "finalize_smem", "committed_smem",
              "prune_wpc", "prune_smem", "prune_wpc_logits", "prune_smem_logits", "n_max")
_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "native", "emulate_plan.cpp")
_OUT = os.path.join(_HERE, "native", "_build", "libctc_emul_plan.so")
_plan_full = None


def _build():
    """Compiles tests/native/emulate_plan.cpp (plan.h as the library compiles it) like tests/emul.py does."""
    os.makedirs(os.path.dirname(_OUT), exist_ok=True)
    csrc = os.path.join(_HERE, "..", "ctcdecode_b200", "csrc")
    deps = [_SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
    if not (os.path.exists(_OUT) and all(os.path.getmtime(_OUT) >= os.path.getmtime(d) for d in deps)):
        tmp = _OUT + ".tmp%d" % os.getpid()
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-nostdlib++", "-Wno-unused-function", _SRC,
                        "-o", tmp, "-l:libstdc++.so.6", "-lm"], check=True)
        os.replace(tmp, _OUT)
    return _OUT


def plan_or_refusal(B, T, V, beam, cutoff_prob=1.0, cutoff_top_n=40, scorer=False):
    """What plan.h decides (scorer: a scorer is attached), through emu_plan_full: (dict of _PLAN_KEYS, None), or
    (CTCDEC_E_* code, the plan's message)."""
    global _plan_full
    if _plan_full is None:
        _plan_full = ctypes.CDLL(_build()).emu_plan_full
        _plan_full.restype = ctypes.c_int
        _plan_full.argtypes = [ctypes.c_int] * 4 + [ctypes.c_double, ctypes.c_int, ctypes.c_int,
                                                    ctypes.POINTER(ctypes.c_int32), ctypes.c_char_p, ctypes.c_int]
    out = (ctypes.c_int32 * len(_PLAN_KEYS))()
    msg = ctypes.create_string_buffer(256)
    rc = _plan_full(B, T, V, beam, cutoff_prob, cutoff_top_n, int(bool(scorer)), out, msg, len(msg))
    if rc:
        return rc, msg.value.decode()
    return dict(zip(_PLAN_KEYS, list(out))), None


def plan_dict(B, T, V, beam, cutoff_prob=1.0, cutoff_top_n=40, scorer=False):
    """plan_or_refusal's dict, or the CTCDEC_E_* code."""
    return plan_or_refusal(B, T, V, beam, cutoff_prob, cutoff_top_n, scorer)[0]


def plan(scorer, batch, mode, V, K):
    return plan_or_refusal(BATCHES[batch], 20, V, K, scorer=scorer, **MODES[mode](V))


def check_layout(pl, V, K, scorer, where):
    """The beam-kernel layout's regions, in the order make_layout (beam_core.cuh) lays them out, each with room for
    what the kernel keeps there, disjoint and inside the CTA's shared memory; then the other kernels' shared memory."""
    KP, W, WC, NW, seg, F, NP = pl["KP"], pl["W"], pl["WC"], pl["NW"], pl["seg"], pl["F"], pl["NP"]
    sorted_ = bool(pl["sorted"])
    assert KP >= K and KP % 32 == 0 and (K <= 256 or KP - K < 32), where
    assert NW * 32 == pl["NT"] and W == (NP + 31) // 32 and WC == (V + 31) // 32, where
    mwords = W if scorer else max(W, WC)
    regions = [  # (offset, bytes the kernel addresses there)
        ("evcnt", pl["evcnt"], KP // 32 * 4),
        ("mask", pl["mask"], KP * mwords * 4),
        ("mask2", pl["mask2"], KP * mwords * 4),
        ("rmask", pl["rmask"], KP * W * 4),
        ("dmask", pl["dmask"], KP * WC * 4 if scorer else 0),
        ("rank", pl["rank"], 2 * ((V * 2 + 15) // 16 * 16) if sorted_ else 0),
        ("tile_lp", pl["tile_lp"], 2 * F * NP * 4),
        ("tile_idx", pl["tile_idx"], 2 * F * NP * 2 if sorted_ else 0),
        ("clk", pl["clk"], NW * seg * 4),
        ("cli", pl["cli"], NW * seg * 4),
    ]
    assert regions[0][1] > 0, where
    for (n0, o0, b0), (n1, o1, _) in zip(regions, regions[1:]):
        assert o0 + b0 <= o1, (where, n0, n1, pl)
    name, o, b = regions[-1]
    assert o + b <= pl["smem"] <= SMEM_CTA, (where, pl)
    assert pl["tile_lp"] % 128 == 0 and pl["clk"] % 16 == 0 and pl["cli"] % 16 == 0, (where, pl)
    assert seg >= 32, (where, pl)
    assert F == 1 or F * NP * 4 <= 4096, (where, pl)   # tiles of one frame once a row passes 4 KB
    assert pl["P"] >= V and pl["P"] & (pl["P"] - 1) == 0, (where, pl)
    assert pl["finalize_smem"] <= SMEM_CTA and pl["committed_smem"] <= SMEM_CTA, (where, pl)
    for wpc, smem in ((pl["prune_wpc"], pl["prune_smem"]), (pl["prune_wpc_logits"], pl["prune_smem_logits"])):
        assert 1 <= wpc <= 8 and smem <= SMEM_CTA, (where, pl)


def check_refusal(res, where):
    rc, msg = res
    assert rc == CTCDEC_E_UNSUPPORTED, (where, res)
    m = re.search(r"needs (\d+) bytes of shared memory", msg)
    if m:
        assert int(m.group(1)) > SMEM_CTA and "227 KB" in msg, (where, msg)
    else:
        assert "vocabulary sort (at most 16384)" in msg, (where, msg)
    return msg


@pytest.mark.parametrize("cell", CELLS, ids=_ids)
def test_largest_beam_per_vocabulary(cell):
    """Every beam in [1, KMAX] is accepted with a layout that fits, every beam above it up to 4096 is refused."""
    scorer, batch, mode = cell
    got = []
    for V, kmax in zip(VOCABS, KMAX[cell]):
        accepted = 0
        for K in list(range(1, kmax + 97)) + [1024, 2048, 4096]:
            pl, msg = plan(scorer, batch, mode, V, K)
            if isinstance(pl, dict):
                assert K == accepted + 1, (cell, V, K, "accepted beams are not one range")
                accepted = K
                check_layout(pl, V, K, scorer, (cell, V, K))
            elif K == kmax + 1:
                check_refusal((pl, msg), (cell, V, K))
        got.append(accepted)
    assert tuple(got) == KMAX[cell], (cell, got)


@pytest.mark.parametrize("cell", CELLS, ids=_ids)
def test_largest_vocabulary_per_beam(cell):
    """Every vocabulary in [1, VMAX] is accepted with a layout that fits, every one above it is refused."""
    scorer, batch, mode = cell
    got = []
    for K, vmax in zip(BEAMS, VMAX[cell]):
        # every vocabulary up to 300 and within 96 of the edge, every 7th in between (all of them take minutes)
        vs = sorted(set(range(1, 301)) | set(range(301, vmax, 7)) | set(range(max(1, vmax - 96), vmax + 97)))
        accepted = 0
        for V in vs + [20000, 32768, 65534]:
            pl, msg = plan(scorer, batch, mode, V, K)
            if isinstance(pl, dict):
                assert V <= vmax, (cell, K, V, "accepted above the edge")
                accepted = V
                check_layout(pl, V, K, scorer, (cell, V, K))
            else:
                assert V > vmax, (cell, K, V, "refused below the edge")
                check_refusal((pl, msg), (cell, V, K))
        got.append(accepted)
    assert tuple(got) == VMAX[cell], (cell, got)


def test_scorer_layout_is_the_one_checked():
    """Shapes whose plain layout fits but whose scorer layout (+ the [KP][WC] dictionary masks) does not: the plan with
    a scorer refuses them, naming the layout size, instead of accepting them for a kernel that cannot launch."""
    for V, K, kw in ((29, 705, dict()), (29, 736, dict()), (256, 544, dict(cutoff_top_n=256)),
                     (1024, 320, dict(cutoff_top_n=1024)), (9054, 1, dict(cutoff_top_n=9054))):
        assert isinstance(plan_dict(8, 20, V, K, **kw), dict), (V, K)
        rc, msg = plan_or_refusal(8, 20, V, K, scorer=True, **kw)
        assert "with a scorer" in check_refusal((rc, msg), (V, K)), msg


def test_scorer_plan_at_one_stream_covers_every_batch():
    """A streaming state with a scorer is checked at creation with a batch of one; every batch it can later be decoded
    in must fit as well (the throughput plan's edges are never below the latency plan's)."""
    for mode in MODES:
        for i, V in enumerate(VOCABS):
            assert KMAX[(True, "throughput", mode)][i] >= KMAX[(True, "latency", mode)][i]
        for i, K in enumerate(BEAMS):
            assert VMAX[(True, "throughput", mode)][i] >= VMAX[(True, "latency", mode)][i]
    for V, K, kw in ((29, 704, {}), (6, 736, dict(cutoff_prob=0.99)), (9053, 8, dict(cutoff_top_n=9053))):
        one = plan_dict(1, 20, V, K, scorer=True, **kw)
        if isinstance(one, dict):
            for B in (2, 264, 265, 300, 4096):
                assert isinstance(plan_dict(B, 20, V, K, scorer=True, **kw), dict), (V, K, B)
