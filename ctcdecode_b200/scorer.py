"""Scorer plumbing for the language-model path.

The language model stays on the host behind the hook of include/ctcdecode_b200.h (``ctcdec_scorer_hooks``); this
package ships no KenLM.  A *provider* is a shared library -- normally the reference's own extension with the
small stub of INTEGRATION.md section 6 -- that owns the real ``Scorer`` (KenLM) and exports:

    void  *ref_scorer_new(double alpha, double beta, const char *lm_path, const char *const *labels, int n)
    void   ref_scorer_free(void *)
    int    ref_scorer_is_character_based(void *)
    size_t ref_scorer_max_order(void *)
    void   ref_scorer_reset_params(void *, double alpha, double beta)
    double ref_scorer_cond_from_labels(void *, const int *labels, int n)   # get_log_cond_prob(make_ngram(prefix))
    double ref_scorer_sent_from_labels(void *, const int *labels, int n)   # get_sent_log_prob(split_labels(prefix))
    size_t ref_lm_vocabulary(const char *lm_path, char *buf, size_t cap)   # '\\n'-separated LM vocabulary

providers/ in this repository holds exactly that stub (kenlm_provider.cpp) and the recipe (Makefile) that builds it
from the reference's sources where they lie: providers/_build/libkenlm_provider.so, used when present.  Another
provider is chosen with ``scorer_provider=`` or the environment variable CTCDECODE_B200_SCORER_PROVIDER.

``scorer_provider="device"`` (or CTCDECODE_B200_SCORER_PROVIDER=device) needs no provider: ``ArpaScorer`` has the
library read the model file itself (ctcdec_scorer_create_arpa): ARPA text, or a KenLM binary file of any type KenLM's
build_binary writes but REST_PROBING (probing, trie, quantized and array-compressed tries; a probing file's tables and
a trie file's packed arrays are searched on the device as they are).  Its hooks reproduce the
reference Scorer over KenLM bit for bit; a model they cannot reproduce exactly (order above 6, REST_PROBING, a damaged
binary, ...) is refused.
"""
import ctypes
import os

from . import _native

DEFAULT_PROVIDER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "providers", "_build",
                                "libkenlm_provider.so")


DEVICE = "device"


def make_scorer(labels, model_path, alpha, beta, provider=None):
    """The scorer for ``model_path``: the library's own ARPA scorer for provider "device", else a provider's."""
    provider = provider or os.environ.get("CTCDECODE_B200_SCORER_PROVIDER")
    if provider == DEVICE:
        return ArpaScorer(labels, model_path, alpha, beta)
    return ProviderScorer(labels, model_path, alpha, beta, provider)


class ArpaScorer(object):
    """The library-side scorer built from an ARPA or KenLM binary file by the library itself (no provider library, no
    KenLM)."""

    def __init__(self, labels, model_path, alpha, beta):
        self.handle = None
        if not os.path.exists(model_path):
            raise FileNotFoundError(model_path)
        self._lib = _native.load()
        labels = list(labels)
        lab = (ctypes.c_char_p * len(labels))(*[s.encode() for s in labels])
        path = model_path.encode() if isinstance(model_path, str) else model_path
        handle = ctypes.c_void_p()
        _native.check(self._lib.ctcdec_scorer_create_arpa(path, float(alpha), float(beta), lab, len(labels),
                                                          ctypes.byref(handle)))
        self.handle = handle.value

    def is_character_based(self):
        return int(self._lib.ctcdec_scorer_is_character_based(self.handle))

    def max_order(self):
        return int(self._lib.ctcdec_scorer_max_order(self.handle))

    def dict_size(self):
        return int(self._lib.ctcdec_scorer_dict_size(self.handle))

    def table_bytes(self):
        """bytes of n-gram data (unigrams and orders >= 2) the model puts in each device's memory"""
        n = ctypes.c_size_t()
        _native.check(self._lib.ctcdec_scorer_table_bytes(self.handle, ctypes.byref(n)))
        return int(n.value)

    def reset_params(self, alpha, beta):
        _native.check(self._lib.ctcdec_scorer_reset_params(self.handle, float(alpha), float(beta)))

    def release(self):
        if getattr(self, "handle", None):
            self._lib.ctcdec_scorer_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class ProviderScorer(object):
    """Owns the provider's Scorer and the library-side scorer object (dictionary on the GPU, hook pointers)."""

    def __init__(self, labels, model_path, alpha, beta, provider=None):
        provider = provider or os.environ.get("CTCDECODE_B200_SCORER_PROVIDER")
        if not provider and os.path.exists(DEFAULT_PROVIDER):
            provider = DEFAULT_PROVIDER  # providers/Makefile: the reference's Scorer + KenLM behind the C-ABI stub
        if not provider:
            raise RuntimeError(
                "ctcdecode_b200: model_path needs a scorer provider library (scorer_provider=... or "
                "CTCDECODE_B200_SCORER_PROVIDER): the language model stays on the host behind the reference's own "
                "Scorer; see INTEGRATION.md section 6")
        if not os.path.exists(model_path):
            raise FileNotFoundError(model_path)
        self._lib = _native.load()
        P = ctypes.CDLL(provider)
        self._P = P
        cpp = ctypes.POINTER(ctypes.c_char_p)
        P.ref_scorer_new.restype = ctypes.c_void_p
        P.ref_scorer_new.argtypes = [ctypes.c_double, ctypes.c_double, ctypes.c_char_p, cpp, ctypes.c_int]
        P.ref_scorer_free.argtypes = [ctypes.c_void_p]
        P.ref_scorer_is_character_based.argtypes = [ctypes.c_void_p]
        P.ref_scorer_max_order.argtypes = [ctypes.c_void_p]
        P.ref_scorer_max_order.restype = ctypes.c_size_t
        P.ref_scorer_reset_params.argtypes = [ctypes.c_void_p, ctypes.c_double, ctypes.c_double]
        P.ref_lm_vocabulary.restype = ctypes.c_size_t
        P.ref_lm_vocabulary.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        labels = list(labels)
        lab = (ctypes.c_char_p * len(labels))(*[s.encode() for s in labels])
        path = model_path.encode() if isinstance(model_path, str) else model_path
        self._ctx = P.ref_scorer_new(float(alpha), float(beta), path, lab, len(labels))
        n = P.ref_lm_vocabulary(path, None, 0)
        buf = ctypes.create_string_buffer(n)
        P.ref_lm_vocabulary(path, buf, n)
        words = buf.value.split(b"\n")[:-1]
        wrd = (ctypes.c_char_p * max(1, len(words)))(*words) if words else (ctypes.c_char_p * 1)()
        hooks = _native.ScorerHooks(self._ctx, ctypes.cast(P.ref_scorer_cond_from_labels, ctypes.c_void_p).value,
                                    ctypes.cast(P.ref_scorer_sent_from_labels, ctypes.c_void_p).value)
        handle = ctypes.c_void_p()
        self.handle = None
        _native.check(self._lib.ctcdec_scorer_create(ctypes.byref(hooks), float(alpha), float(beta), lab, len(labels),
                                                     wrd, len(words), int(P.ref_scorer_max_order(self._ctx)),
                                                     int(P.ref_scorer_is_character_based(self._ctx)),
                                                     ctypes.byref(handle)))
        self.handle = handle.value

    def is_character_based(self):
        return int(self._lib.ctcdec_scorer_is_character_based(self.handle))

    def max_order(self):
        return int(self._lib.ctcdec_scorer_max_order(self.handle))

    def dict_size(self):
        return int(self._lib.ctcdec_scorer_dict_size(self.handle))

    def reset_params(self, alpha, beta):
        self._P.ref_scorer_reset_params(self._ctx, float(alpha), float(beta))
        _native.check(self._lib.ctcdec_scorer_reset_params(self.handle, float(alpha), float(beta)))

    def release(self):
        if getattr(self, "handle", None):
            self._lib.ctcdec_scorer_destroy(self.handle)
            self.handle = None
        if getattr(self, "_ctx", None):
            self._P.ref_scorer_free(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass
