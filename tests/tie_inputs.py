"""Seeded inputs on which the reference's unspecified tie resolution matters, and rows of degenerate values, for the
parity tests that compare against every output the reference may produce (oracle.CPort.decode_alternatives)."""
import numpy as np

from oracle.oracle import result_key

FLT_MAX = float(np.finfo(np.float32).max)

# degenerate_probs() kinds: probability input first, then log-probability input
DEGENERATE = ("zeros", "subnormal", "above_one", "onehot_blank", "log_zeros", "log_extremes", "blank_neg_inf")

# one decoder configuration per path of the vocabulary cut (prune_program.cuh): V, decoder arguments
PRUNE_PATHS = {
    "index_v29": (29, dict(beam=16)),                                  # index order, V <= 32
    "index_wide_v100": (100, dict(beam=16, cutoff_top_n=100)),         # index order, wide-row loop
    "top_select_v64": (64, dict(beam=16, cutoff_top_n=12)),            # partial top_select, V <= 64
    "top_select_equal_v256": (256, dict(beam=16, cutoff_top_n=40)),    # > 64 keys equal to the cut value
    "bitonic_v1500": (1500, dict(beam=8, cutoff_top_n=40)),            # full bitonic sort
    "cutoff_prob_v64": (64, dict(beam=16, cutoff_prob=0.99)),          # fp64 cutoff_prob chain
}


def _softmax_rows(rng, B, T, V, blank_id):
    x = 2.0 * rng.randn(B, T, V)
    x[:, :, blank_id] += 3.0 * (rng.rand(B, T) < 0.6)
    e = np.exp(x - x.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _zero_out(rng, p):
    """Exact zeros: per frame between half and all but one of the entries.  With V = 256 and top-n 40 the cut then
    often falls inside a block of more than 64 equal (zero) keys."""
    B, T, V = p.shape
    for b in range(B):
        for t in range(T):
            k = rng.randint(V // 2, V)
            p[b, t, rng.permutation(V)[:k]] = 0.0
    return p


def degenerate_probs(kind, B, T, V, seed, blank_id=0):
    """Returns (float32 [B, T, V], log_input) for one DEGENERATE kind."""
    rng = np.random.RandomState(seed)
    p = _softmax_rows(rng, B, T, V, blank_id)
    if kind == "zeros":
        return _zero_out(rng, p).astype(np.float32), False
    if kind == "subnormal":                     # a third of the entries subnormal (float32 < 1.18e-38)
        p = p.astype(np.float32)
        m = rng.rand(B, T, V) < 1 / 3
        p[m] = rng.uniform(1e-45, 1e-39, size=int(m.sum())).astype(np.float32)
        return p, False
    if kind == "above_one":                     # rows that sum to 1.5 .. 40, entries up to 40
        return (p * rng.choice([1.5, 3.0, 40.0], size=(B, T, 1))).astype(np.float32), False
    if kind == "onehot_blank":                  # every other frame is blank with near-certainty: tiny off-peak values,
        for b in range(B):                      # distinct within the frame and from frame to frame
            for t in range(0, T, 2):            # (exact-zero off-peak values are the "zeros" kind)
                p[b, t] = 1e-30 * rng.uniform(1.0, 2.0, size=V)
                p[b, t, blank_id] = 1.0
        return p.astype(np.float32), False
    if kind == "log_zeros":                     # torch.log of rows with zeros: -inf entries
        with np.errstate(divide="ignore"):
            return np.log(_zero_out(rng, p).astype(np.float32)), True
    if kind == "log_extremes":                  # -FLT_MAX, -1e30, positive and large log-probabilities
        lp = np.log(p).astype(np.float32)
        u = rng.rand(B, T, V)
        lp[u < 0.1] = -FLT_MAX
        lp[(u >= 0.1) & (u < 0.2)] = -1e30
        pos = (u >= 0.2) & (u < 0.22)
        lp[pos] = rng.uniform(0.0, 20.0, size=int(pos.sum())).astype(np.float32)
        lp[u >= 0.995] = 1e4
        return lp, True
    if kind == "blank_neg_inf":                 # blank impossible for whole stretches of 8 frames
        lp = np.log(p).astype(np.float32)
        for t in range(T):
            if (t // 8) % 2:
                lp[:, t, blank_id] = -np.inf
        return lp, True
    raise ValueError(kind)


def quantised_probs(B, T, V, seed, levels=(1.0, 2.0, 4.0)):
    """Rows whose entries take a few distinct values, normalised: equal log-probabilities everywhere, so equal prefix
    scores -- and comparator-equal prefixes straddling the beam cut (TIE_PRUNE) -- are common."""
    rng = np.random.RandomState(seed)
    p = np.asarray(levels, np.float32)[rng.randint(0, len(levels), size=(B, T, V))]
    return (p / p.sum(-1, keepdims=True)).astype(np.float32)


def resolved_by_alternative(ref, got):
    """Utterances that equal one of the reference's permitted outputs but NOT the oracle's default resolution (after
    compare() has passed): the count of ties whose resolution the default could not have checked."""
    n = 0
    for b in range(ref["lens"].shape[0]):
        if not ref["unresolved"][b] and len(ref["alternatives"][b]) > 1:
            n += result_key(got, b) != result_key(ref["alternatives"][b][0])
    return n
