"""TEST INFRASTRUCTURE ONLY -- ctypes front-ends to the two CPU checkers.

* ``CPort``      -> oracle/libctc_oracle.so, the plain-C restatement (oracle/ctc_oracle.c).
* ``Reference``  -> oracle/_ref/libctcref.so, the UNMODIFIED reference sources compiled by
                    oracle/Makefile behind the C-ABI driver oracle/ref_capi.cpp (needs
                    /root/reference at build time only; the built .so travels to the GPU box).

Both return numpy arrays shaped like the reference's tensors (reference __init__.py:83-86):
tokens/timesteps int32 [B, beam, T] (only [:len] meaningful -- here the rest is filled with -1
instead of being left uninitialised), scores float32 [B, beam], lens int32 [B, beam], plus
n_results int32 [B].
"""
import ctypes
import math
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_i32p = ctypes.POINTER(ctypes.c_int32)
_f32p = ctypes.POINTER(ctypes.c_float)


def _p(a, t):
    return a.ctypes.data_as(t)


def build(ref=True):
    """Compile the C port and (when /root/reference is present) the reference build."""
    subprocess.run(["make", "-s", "-C", _HERE, "libctc_oracle.so"], check=True)
    if ref and os.path.isdir(os.environ.get("CTC_REFERENCE_DIR", "/root/reference")):
        subprocess.run(["make", "-s", "-j8", "-C", _HERE, "ref"], check=True)


def _alloc(B, beam, T):
    return (np.full((B, beam, T), -1, np.int32), np.full((B, beam, T), -1, np.int32),
            np.zeros((B, beam), np.float32), np.zeros((B, beam), np.int32), np.zeros((B,), np.int32))


def _prep(probs, seq_lens):
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    B, T, V = probs.shape
    if seq_lens is None:
        seq_lens = np.full((B,), T, np.int32)
    seq_lens = np.ascontiguousarray(seq_lens, dtype=np.int32)
    return probs, seq_lens, B, T, V


TIE_PRUNE, TIE_FINAL, TIE_VOCAB = 1, 2, 4   # tie_flags bits (ctc_oracle.c)


def result_key(d, b=0):
    """Hashable form of utterance b of a result dict: n_results and its rows (score bits, len, tokens, timesteps), rows
    inside a run of equal (score bits, last token) sorted -- the reference's final sort may emit those in any order."""
    n = int(d["n_results"][b])
    rows = []
    for p in range(n):
        L = int(d["lens"][b, p])
        rows.append((int(d["scores"][b, p:p + 1].view(np.int32)[0]), L, tuple(d["tokens"][b, p, :L].tolist()),
                     tuple(d["timesteps"][b, p, :L].tolist())))
    last = [r[2][-1] if r[1] else -1 for r in rows]
    out, p = [], 0
    while p < n:
        q = p + 1
        while q < n and rows[q][0] == rows[p][0] and last[q] == last[p]:
            q += 1
        out.extend(sorted(rows[p:q]))
        p = q
    return n, tuple(out)


class CPort:
    """The plain-C restatement (no LM)."""

    def __init__(self, path=None):
        path = path or os.path.join(_HERE, "libctc_oracle.so")
        if not os.path.exists(path):
            build(ref=False)
        self.lib = ctypes.CDLL(path)
        L = self.lib
        L.ctc_oracle_decode_batch.restype = ctypes.c_int
        L.ctc_oracle_decode_batch.argtypes = [_f32p, _i32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              _i32p, _i32p, _f32p, _i32p, _i32p, _i32p]
        L.ctc_oracle_decode_choices.restype = ctypes.c_int
        L.ctc_oracle_decode_choices.argtypes = [_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_void_p, ctypes.c_int, _i32p, ctypes.c_int, _i32p, _i32p,
                                                _i32p, _f32p, _i32p, _i32p]
        L.ctc_oracle_state_new.restype = ctypes.c_void_p
        L.ctc_oracle_state_new.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int]
        L.ctc_oracle_state_free.argtypes = [ctypes.c_void_p]
        L.ctc_oracle_state_next.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_int]
        L.ctc_oracle_state_decode.restype = ctypes.c_int
        L.ctc_oracle_state_decode.argtypes = [ctypes.c_void_p, ctypes.c_int, _i32p, _i32p, _f32p, _i32p, _i32p]
        for name in ("expf", "logf", "logprob"):
            f = getattr(L, "ctc_oracle_%s_array" % name)
            f.argtypes = [_f32p, _f32p, ctypes.c_long]
        L.ctc_oracle_lse_array.argtypes = [_f32p, _f32p, _f32p, ctypes.c_long]
        L.ctc_oracle_f64_array.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long]

    def decode(self, probs, seq_lens=None, beam=100, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0,
               log_input=False):
        probs, seq_lens, B, T, V = _prep(probs, seq_lens)
        tok, ts, sc, ln, nres = _alloc(B, beam, T)
        ties = np.zeros((B,), np.int32)
        self.lib.ctc_oracle_decode_batch(_p(probs, _f32p), _p(seq_lens, _i32p), B, T, V, beam, cutoff_prob,
                                         cutoff_top_n, blank_id, int(log_input), _p(tok, _i32p), _p(ts, _i32p),
                                         _p(sc, _f32p), _p(ln, _i32p), _p(nres, _i32p), _p(ties, _i32p))
        return dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, n_results=nres, ties=ties)

    def decode_choices(self, row, length, choices=(), beam=100, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0,
                       log_input=False):
        """One utterance (row: [T, V]) with the beam-cut tie choices `choices` (see ctc_oracle_decode_choices; missing
        ones are 0, which is decode()'s resolution).  Returns (result dict shaped like decode()'s for B = 1, events):
        events is an int32 [n, 4] array of (frame, m, r, junk), one row per tie event met."""
        row = np.ascontiguousarray(row, dtype=np.float32)
        T, V = row.shape
        tok, ts, sc, ln, _ = _alloc(1, beam, T)
        ch = np.ascontiguousarray(choices, dtype=np.int64)
        ev = np.zeros((max(T, 1), 4), np.int32)    # at most one tie event per frame
        n_ev, tie = ctypes.c_int(0), ctypes.c_int(0)
        n = self.lib.ctc_oracle_decode_choices(_p(row, _f32p), int(length), T, V, beam, cutoff_prob, cutoff_top_n,
                                               blank_id, int(log_input), ch.ctypes.data, len(ch), _p(ev, _i32p),
                                               ev.shape[0], ctypes.byref(n_ev), _p(tok, _i32p), _p(ts, _i32p),
                                               _p(sc, _f32p), _p(ln, _i32p), ctypes.byref(tie))
        out = dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, n_results=np.array([n], np.int32),
                   ties=np.array([tie.value], np.int32))
        return out, ev[:n_ev.value]

    def _enumerate(self, row, length, cap, kw):
        """Depth-first walk over the choice vectors of one utterance: every leaf is one complete decode.  Returns (the
        distinct outputs, the choice-0 decode first; unresolved; junk).  Unresolved: a tie among -FLT_MAX "junk"
        prefixes (SURVEY.md quirk Q6; their groups are far too large to enumerate -- `junk` is then set) or more than
        `cap` leaves."""
        alts, seen, leaves = [], set(), 0
        stack = [()]
        while stack:
            choices = stack.pop()
            out, events = self.decode_choices(row, length, choices, **kw)
            leaves += 1
            if events[:, 3].any():
                return alts or [out], True, True
            key = result_key(out)
            if key not in seen:
                seen.add(key)
                alts.append(out)
            # branch at every event this run took the default for: events before len(choices) are fixed by `choices`
            for j in range(len(events) - 1, len(choices) - 1, -1):
                k = math.comb(int(events[j, 1]), int(events[j, 2]))
                if leaves + len(stack) + k - 1 > cap:
                    return alts, True, False
                pad = choices + (0,) * (j - len(choices))
                stack.extend(pad + (c,) for c in range(k - 1, 0, -1))
        return alts, False, False

    def decode_alternatives(self, probs, seq_lens=None, cap=64, beam=100, cutoff_prob=1.0, cutoff_top_n=40,
                            blank_id=0, log_input=False, threads=None):
        """decode(), plus every output the reference may produce where it is unspecified.  At a beam-cut tie
        (TIE_PRUNE) the reference keeps some r of the m comparator-equal prefixes straddling the cut; for each
        TIE_PRUNE-flagged utterance every combination of such choices is decoded.  Adds to decode()'s dict:
          alternatives[b]  list of distinct B = 1 result dicts (alternatives[b][0] is decode()'s own row);
          unresolved[b]    bool: junk ties or more than `cap` choice vectors -- the list is then incomplete;
          junk_ties[b]     bool: unresolved because a tie among -FLT_MAX junk prefixes was met.
        Distinct means: tokens, timesteps, score bits, lens and n_results differ after rows of equal (score, last
        token) -- which the reference's final sort may emit in either order (TIE_FINAL) -- are put in canonical order.
        Flagged utterances are enumerated on `threads` threads (the C calls release the GIL)."""
        kw = dict(beam=beam, cutoff_prob=cutoff_prob, cutoff_top_n=cutoff_top_n, blank_id=blank_id, log_input=log_input)
        base = self.decode(probs, seq_lens, **kw)
        probs, seq_lens, B, T, V = _prep(probs, seq_lens)
        alts = [[{k: v[b:b + 1] for k, v in base.items()}] for b in range(B)]
        unresolved, junk = np.zeros((B,), bool), np.zeros((B,), bool)
        todo = [b for b in range(B) if base["ties"][b] & TIE_PRUNE]
        if todo:
            with ThreadPoolExecutor(threads or len(os.sched_getaffinity(0))) as ex:
                for b, res in zip(todo, ex.map(lambda b: self._enumerate(probs[b], seq_lens[b], cap, kw), todo)):
                    alts[b], unresolved[b], junk[b] = res
        base["alternatives"] = alts
        base["unresolved"] = unresolved
        base["junk_ties"] = junk
        return base

    # --- streaming (mirrors DecoderState next()/decode()) ---
    def state_new(self, V, beam, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0, log_input=False):
        return self.lib.ctc_oracle_state_new(V, beam, cutoff_prob, cutoff_top_n, blank_id, int(log_input))

    def state_next(self, st, chunk):
        chunk = np.ascontiguousarray(chunk, dtype=np.float32)
        self.lib.ctc_oracle_state_next(st, _p(chunk, _f32p), chunk.shape[0])

    def state_decode(self, st, beam, max_len):
        tok = np.full((beam, max_len), -1, np.int32)
        ts = np.full((beam, max_len), -1, np.int32)
        sc = np.zeros((beam,), np.float32)
        ln = np.zeros((beam,), np.int32)
        tie = ctypes.c_int(0)
        n = self.lib.ctc_oracle_state_decode(st, max_len, _p(tok, _i32p), _p(ts, _i32p), _p(sc, _f32p),
                                             _p(ln, _i32p), ctypes.byref(tie))
        return dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, n_results=n, ties=tie.value)

    def state_free(self, st):
        self.lib.ctc_oracle_state_free(st)

    # --- libm probes ---
    def _map(self, name, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        getattr(self.lib, "ctc_oracle_%s_array" % name)(_p(x, _f32p), _p(y, _f32p), x.size)
        return y

    def expf(self, x):
        return self._map("expf", x)

    def logf(self, x):
        return self._map("logf", x)

    def logprob(self, p):
        return self._map("logprob", p)

    def lse(self, x, y):
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.ascontiguousarray(y, dtype=np.float32)
        z = np.empty_like(x)
        self.lib.ctc_oracle_lse_array(_p(x, _f32p), _p(y, _f32p), _p(z, _f32p), x.size)
        return z


    def f64(self, which, x, x2=None):
        """host libm in double: which 0 exp(x), 1 log(x), 2 log_sum_exp<double>(x, x2)"""
        x = np.ascontiguousarray(x, dtype=np.float64)
        x2 = None if x2 is None else np.ascontiguousarray(x2, dtype=np.float64)
        y = np.empty_like(x)
        self.lib.ctc_oracle_f64_array(which, x.ctypes.data, None if x2 is None else x2.ctypes.data, y.ctypes.data, x.size)
        return y


# scorer provider built from the reference's Scorer + KenLM (oracle/Makefile `provider`): the language-model hook
PROVIDER = os.path.join(_HERE, "_ref", "provider", "libkenlm_provider.so")


def reference_available():
    return os.path.exists(os.path.join(_HERE, "_ref", "libctcref.so"))


class Reference:
    """The unmodified reference C++ (ThreadPool batch path), optional KenLM scorer."""

    def __init__(self, labels, model_path=None, alpha=0.0, beta=0.0, path=None):
        path = path or os.path.join(_HERE, "_ref", "libctcref.so")
        self.lib = ctypes.CDLL(path)
        L = self.lib
        self.labels = list(labels)
        self._labels_c = (ctypes.c_char_p * len(self.labels))(*[s.encode() for s in self.labels])
        cpp = ctypes.POINTER(ctypes.c_char_p)
        L.ref_scorer_new.restype = ctypes.c_void_p
        L.ref_scorer_new.argtypes = [ctypes.c_double, ctypes.c_double, ctypes.c_char_p, cpp, ctypes.c_int]
        L.ref_scorer_free.argtypes = [ctypes.c_void_p]
        L.ref_scorer_is_character_based.argtypes = [ctypes.c_void_p]
        L.ref_scorer_max_order.argtypes = [ctypes.c_void_p]
        L.ref_scorer_max_order.restype = ctypes.c_size_t
        L.ref_scorer_dict_size.argtypes = [ctypes.c_void_p]
        L.ref_scorer_dict_size.restype = ctypes.c_size_t
        L.ref_scorer_reset_params.argtypes = [ctypes.c_void_p, ctypes.c_double, ctypes.c_double]
        L.ref_decode_batch.restype = ctypes.c_int
        L.ref_decode_batch.argtypes = [_f32p, _i32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, cpp, ctypes.c_size_t,
                                       ctypes.c_size_t, ctypes.c_double, ctypes.c_size_t, ctypes.c_size_t,
                                       ctypes.c_int, ctypes.c_void_p, _i32p, _i32p, _f32p, _i32p, _i32p]
        L.ref_state_new.restype = ctypes.c_void_p
        L.ref_state_new.argtypes = [cpp, ctypes.c_int, ctypes.c_size_t, ctypes.c_double, ctypes.c_size_t,
                                    ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
        L.ref_state_free.argtypes = [ctypes.c_void_p]
        L.ref_decode_with_states.restype = ctypes.c_int
        L.ref_decode_with_states.argtypes = [_f32p, _i32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_size_t,
                                             ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_uint8),
                                             ctypes.c_int, ctypes.c_int, _i32p, _i32p, _f32p, _i32p, ctypes.c_int,
                                             _i32p]
        L.ref_scorer_cond_from_labels.restype = ctypes.c_double
        L.ref_scorer_cond_from_labels.argtypes = [ctypes.c_void_p, _i32p, ctypes.c_int]
        L.ref_scorer_sent_from_labels.restype = ctypes.c_double
        L.ref_scorer_sent_from_labels.argtypes = [ctypes.c_void_p, _i32p, ctypes.c_int]
        L.ref_lm_vocabulary.restype = ctypes.c_size_t
        L.ref_lm_vocabulary.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        self.scorer = None
        self.model_path = model_path
        if model_path:
            self.scorer = L.ref_scorer_new(alpha, beta, model_path.encode(), self._labels_c, len(self.labels))

    def lm_vocabulary(self):
        """The LM's vocabulary as KenLM enumerates it (what the reference's Scorer::load_lm collects)."""
        n = self.lib.ref_lm_vocabulary(self.model_path.encode(), None, 0)
        buf = ctypes.create_string_buffer(n)
        self.lib.ref_lm_vocabulary(self.model_path.encode(), buf, n)
        return buf.value.decode().split("\n")[:-1]

    def max_order(self):
        return int(self.lib.ref_scorer_max_order(self.scorer))

    def dict_size(self):
        return int(self.lib.ref_scorer_dict_size(self.scorer))

    def is_character_based(self):
        return int(self.lib.ref_scorer_is_character_based(self.scorer))

    def __del__(self):
        if getattr(self, "scorer", None):
            self.lib.ref_scorer_free(self.scorer)
            self.scorer = None

    def decode(self, probs, seq_lens=None, beam=100, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0,
               log_input=False, num_processes=None):
        probs, seq_lens, B, T, V = _prep(probs, seq_lens)
        assert V == len(self.labels)
        if num_processes is None:
            num_processes = len(os.sched_getaffinity(0))
        tok, ts, sc, ln, nres = _alloc(B, beam, T)
        self.lib.ref_decode_batch(_p(probs, _f32p), _p(seq_lens, _i32p), B, T, V, self._labels_c, beam,
                                  num_processes, cutoff_prob, cutoff_top_n, blank_id, int(log_input), self.scorer,
                                  _p(tok, _i32p), _p(ts, _i32p), _p(sc, _f32p), _p(ln, _i32p), _p(nres, _i32p))
        return dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, n_results=nres)

    # --- streaming ---
    def state_new(self, beam, cutoff_prob=1.0, cutoff_top_n=40, blank_id=0, log_input=False):
        return self.lib.ref_state_new(self._labels_c, len(self.labels), beam, cutoff_prob, cutoff_top_n, blank_id,
                                      int(log_input), self.scorer)

    def state_free(self, st):
        self.lib.ref_state_free(st)

    def decode_with_states(self, probs, states, is_eos, beam, seq_lens=None, num_processes=4, max_len=None):
        probs, seq_lens, B, T, V = _prep(probs, seq_lens)
        max_len = max_len or 4096
        tok = np.full((B, beam, max_len), -1, np.int32)
        ts = np.full((B, beam, max_len), -1, np.int32)
        sc = np.zeros((B, beam), np.float32)
        ln = np.zeros((B, beam), np.int32)
        dims = np.zeros((2,), np.int32)
        st = (ctypes.c_void_p * B)(*states)
        eos = (ctypes.c_uint8 * B)(*[1 if e else 0 for e in is_eos])
        rc = self.lib.ref_decode_with_states(_p(probs, _f32p), _p(seq_lens, _i32p), B, T, V, num_processes, st, eos,
                                             beam, max_len, _p(tok, _i32p), _p(ts, _i32p), _p(sc, _f32p),
                                             _p(ln, _i32p), beam, _p(dims, _i32p))
        assert rc == 1, "result larger than max_len cap"
        return dict(tokens=tok, timesteps=ts, scores=sc, lens=ln, dims=dims)
