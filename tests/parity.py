"""Shared comparison helper: bit-exact check of two decoder outputs (dicts of numpy arrays as returned by
oracle.oracle / tests.emul / the CUDA path), honouring the reference's "unspecified" cases.

Integer outputs (tokens, timesteps, lens, n_results) must be identical on [:len]; scores must be identical
as float32 bit patterns (stronger than the 1e-4 the spec asks for).  Beams with score == FLT_MAX are -FLT_MAX "junk"
prefixes (SURVEY.md quirk Q6) whose relative order is a tie by construction: only their pattern is compared.  A tie
in the FINAL order (two result rows with the same score and the same last character, which std::sort may emit in
either order) is compared row-set-wise inside each tied group -- everything else about the utterance must still match.

A tie at a CUT (the beam prune, TIE_PRUNE; the vocabulary prune, TIE_VOCAB) lets the reference keep either of two
equally ranked prefixes.  How compare() treats such an utterance depends on the reference it is given:

* ``ref`` from ``CPort.decode_alternatives`` (the C oracle, which can be steered through its beam-cut ties): every
  output the reference may produce at those ties is known, and ``got`` must equal one of them under the rules above.
  TIE_VOCAB is compared exactly against the oracle's fixed resolution (lowest indices, which the CUDA program keeps
  too); the reference's unstable std::sort may keep other indices there, which is not enumerated.  Only utterances the
  enumerator marks "unresolved" fall back to comparing n_results -- ties among -FLT_MAX junk prefixes, whose groups are
  far too large to enumerate, and utterances whose choice vectors exceed ``cap`` (tie frames chaining on inputs built
  to tie); compare() returns them as its second count.
* any other ``ref`` (a plain decode, the unmodified reference build, the golden fixtures): utterances whose tie flags
  show a cut tie on either side are "skipped" -- only n_results is asserted.
"""
import numpy as np

FLT_MAX = np.float32(3.4028235e38)
_KEYS = ("tokens", "timesteps", "scores", "lens", "n_results", "ties")


def _canonicalise(d, b):
    """Sort rows of utterance b inside every run of equal (score bits, last token) by (tokens, timesteps)."""
    n = int(d["n_results"][b])
    sc = d["scores"][b, :n].view(np.int32)
    lens = d["lens"][b, :n]
    last = np.array([d["tokens"][b, p, lens[p] - 1] if lens[p] > 0 else -1 for p in range(n)])
    p = 0
    while p < n:
        q = p + 1
        while q < n and sc[q] == sc[p] and last[q] == last[p]:
            q += 1
        if q - p > 1:
            rows = list(range(p, q))
            keyf = lambda r: (int(lens[r]), tuple(d["tokens"][b, r, :lens[r]]), tuple(d["timesteps"][b, r, :lens[r]]))  # noqa: E731
            order = sorted(rows, key=keyf)
            for key in ("tokens", "timesteps", "scores", "lens"):
                d[key][b, p:q] = d[key][b, order]
            lens = d["lens"][b, :n]
        p = q


def _row(d, b, p):
    L = int(d["lens"][b, p])
    return (int(d["scores"][b, p:p + 1].view(np.int32)[0]), L, tuple(d["tokens"][b, p, :L]), tuple(d["timesteps"][b, p, :L]))


def _align_permuted_runs(ref, got, b):
    n = int(ref["n_results"][b])
    if int(got["n_results"][b]) != n:
        return
    rr = [_row(ref, b, p) for p in range(n)]
    gr = [_row(got, b, p) for p in range(n)]
    p = 0
    while p < n:
        if rr[p] == gr[p]:
            p += 1
            continue
        q = p
        while q < n and rr[q] != gr[q]:
            q += 1
        if sorted(rr[p:q]) == sorted(gr[p:q]):  # same rows, permuted: give `got` the reference's order
            order = [p + gr[p:q].index(r) for r in rr[p:q]]
            for key in ("tokens", "timesteps", "scores", "lens"):
                got[key][b, p:q] = got[key][b, order]
        p = q


def _utterance(d, b):
    return {k: d[k][b:b + 1] for k in _KEYS if k in d}


def _compare_alternatives(ref, got, name):
    checked, unresolved = 0, 0
    for b in range(ref["lens"].shape[0]):
        if ref["unresolved"][b]:
            unresolved += 1
            assert int(got["n_results"][b]) == int(ref["n_results"][b]), f"{name} utt {b} (unresolved): n_results differ"
            continue
        one = _utterance(got, b)
        got_final = int(one["ties"][0]) & 2 if "ties" in one else 0
        alts = ref["alternatives"][b]
        first_error = None
        for alt in alts:
            try:
                _compare_exact(alt, one, 0, (int(alt["ties"][0]) & 2) | got_final, name)
                break
            except AssertionError as e:
                first_error = first_error or e
        else:
            raise AssertionError(f"{name} utt {b}: equals none of the {len(alts)} outputs the reference may produce; "
                                 f"against the first: {first_error}")
        checked += 1
    return checked, unresolved


def _compare_exact(ref, got, b, final_tie, name):
    if final_tie:  # FLAG_TIE_FINAL: canonical order inside groups of equal (score, last char)
        ref = dict(ref)
        got = dict(got)
        for d in (ref, got):
            for key in ("tokens", "timesteps", "scores", "lens"):
                d[key] = d[key].copy()
            _canonicalise(d, b)
        # With a scorer the tied rows cannot be told from the REPORTED scores (the order is by the raw prefix score,
        # the reported score is the LM-corrected one, reference :187-208): every maximal run of rows that differ
        # must then hold the same rows on both sides, in any order.
        _align_permuted_runs(ref, got, b)
    n = int(ref["n_results"][b])
    assert int(got["n_results"][b]) == n, f"{name} utt {b}: n_results {got['n_results'][b]} != {n}"
    rs, gs = ref["scores"][b, :n], got["scores"][b, :n]
    junk = rs == FLT_MAX
    assert np.array_equal(junk, gs == FLT_MAX), f"{name} utt {b}: junk beam pattern differs"
    ok = ~junk
    assert np.array_equal(rs[ok].view(np.int32), gs[ok].view(np.int32)), \
        f"{name} utt {b}: scores differ\n{rs[ok][:8]}\n{gs[ok][:8]}"
    assert np.array_equal(ref["lens"][b, :n][ok], got["lens"][b, :n][ok]), f"{name} utt {b}: lens differ"
    for p in range(n):
        if junk[p]:
            continue
        L = int(ref["lens"][b, p])
        assert np.array_equal(ref["tokens"][b, p, :L], got["tokens"][b, p, :L]), \
            f"{name} utt {b} beam {p}: tokens differ\n{ref['tokens'][b, p, :L]}\n{got['tokens'][b, p, :L]}"
        assert np.array_equal(ref["timesteps"][b, p, :L], got["timesteps"][b, p, :L]), \
            f"{name} utt {b} beam {p}: timesteps differ\n{ref['timesteps'][b, p, :L]}\n{got['timesteps'][b, p, :L]}"


def compare(ref, got, ref_ties=None, name=""):
    """Asserts parity utterance by utterance; returns (checked, skipped).  With a ``ref`` from
    CPort.decode_alternatives the second count is the number of unresolved utterances (see the module docstring)."""
    if "alternatives" in ref:
        return _compare_alternatives(ref, got, name)
    skipped, checked = 0, 0
    for b in range(ref["lens"].shape[0]):
        tie = 0
        if ref_ties is not None:
            tie |= int(ref_ties[b])
        if "ties" in got:
            tie |= int(got["ties"][b]) & 7
        if tie & 5:  # FLAG_TIE_PRUNE | FLAG_TIE_VOCAB
            # the reference's own choice between comparator-equal prefixes is unspecified here: rows may name different
            # (equally scored) prefixes, and -- the two can split their score differently into blank / non-blank parts
            # -- later scores may differ too.  Only the number of results is asserted; count() below reports how often
            # the multiset of scores and the best beam still agree (tools/tie_report.py: always, on BASELINE configs 2
            # and 4 against oracle/_ref).
            skipped += 1
            assert int(got["n_results"][b]) == int(ref["n_results"][b]), f"{name} utt {b} (tie-flagged): n_results differ"
            continue
        _compare_exact(ref, got, b, tie & 2, name)
        checked += 1
    return checked, skipped


def count(ref, got, ties=None, n=None):
    """Like compare(), but counts instead of asserting: over the first n utterances returns dict(checked, mismatches,
    skipped, tie_prune, tie_vocab, tie_final).  `ties`: flags of either side (the CUDA path's own flags will do: it
    flags exactly the utterances the oracle flags, which the tests assert)."""
    B = ref["lens"].shape[0] if n is None else n
    out = dict(checked=0, mismatches=0, skipped=0, tie_prune=0, tie_vocab=0, tie_final=0, skipped_same_scores=0,
               skipped_same_best_beam=0)
    for b in range(B):
        tie = int(ties[b]) & 7 if ties is not None else 0
        if "ties" in got:
            tie |= int(got["ties"][b]) & 7
        out["tie_prune"] += 1 if tie & 1 else 0
        out["tie_vocab"] += 1 if tie & 4 else 0
        out["tie_final"] += 1 if tie & 2 else 0
        one_ref = {k: v[b:b + 1] for k, v in ref.items() if hasattr(v, "shape") and v.shape[:1] == ref["lens"].shape[:1]}
        one_got = {k: v[b:b + 1] for k, v in got.items() if hasattr(v, "shape") and v.shape[:1] == got["lens"].shape[:1]}
        if tie & 5:  # what the skipped utterances still have in common with the reference
            nr = int(ref["n_results"][b])
            if int(got["n_results"][b]) == nr:
                rs, gs = ref["scores"][b, :nr].view(np.int32), got["scores"][b, :nr].view(np.int32)
                out["skipped_same_scores"] += int(np.array_equal(np.sort(rs), np.sort(gs)))
                L = int(ref["lens"][b, 0]) if nr else 0
                out["skipped_same_best_beam"] += int(nr > 0 and int(got["lens"][b, 0]) == L and
                                                     np.array_equal(ref["tokens"][b, 0, :L], got["tokens"][b, 0, :L]))
        try:
            c, s = compare(one_ref, one_got, [tie], "utt %d" % b)
            out["checked"] += c
            out["skipped"] += s
        except AssertionError:
            out["checked"] += 1
            out["mismatches"] += 1
    return out
