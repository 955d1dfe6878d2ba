"""ctypes binding of include/ctcdecode_b200.h.  Fails loudly: there is no CPU or PyTorch fallback."""
import ctypes
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
# (CTCDECODE_B200_LIB: another build of the same ABI, for A/B measurements of kernel variants)
LIB_PATH = os.environ.get("CTCDECODE_B200_LIB") or os.path.join(_PKG, "_lib", "libctcdecode_b200.so")

OK = 0
FLAG_TIE_PRUNE, FLAG_TIE_FINAL, FLAG_TIE_VOCAB, FLAG_ERR_ARENA = 1, 2, 4, 256


class Config(ctypes.Structure):
    _fields_ = [("vocab_size", ctypes.c_int), ("beam_size", ctypes.c_int), ("blank_id", ctypes.c_int),
                ("log_input", ctypes.c_int), ("cutoff_top_n", ctypes.c_int), ("cutoff_prob", ctypes.c_double)]


class ScorerHooks(ctypes.Structure):
    """ctcdec_scorer_hooks: raw C function pointers (addresses) supplied by the integrator."""
    _fields_ = [("ctx", ctypes.c_void_p), ("cond_log_prob", ctypes.c_void_p), ("sent_log_prob", ctypes.c_void_p)]


class NativeError(RuntimeError):
    pass


_vp = ctypes.c_void_p
_SIGNATURES = {
    "ctcdec_version": (ctypes.c_char_p, []),
    "ctcdec_last_error": (ctypes.c_char_p, []),
    "ctcdec_device_count": (ctypes.c_int, []),
    "ctcdec_workspace_bytes": (ctypes.c_int, [ctypes.POINTER(Config), ctypes.c_int, ctypes.c_int,
                                              ctypes.POINTER(ctypes.c_size_t)]),
    "ctcdec_decode_batch_device": (ctypes.c_int, [ctypes.POINTER(Config), _vp, _vp, ctypes.c_int, ctypes.c_int,
                                                  _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_size_t, _vp]),
    "ctcdec_decode_batch_device_logits": (ctypes.c_int, [ctypes.POINTER(Config), _vp, ctypes.c_int, _vp, ctypes.c_int,
                                                         ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                                         ctypes.c_size_t, _vp]),
    "ctcdec_pack_results_device": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp,
                                                  _vp, _vp, ctypes.c_size_t, _vp]),
    "ctcdec_decode_batch_host": (ctypes.c_int, [ctypes.POINTER(Config), _vp, _vp, ctypes.c_int, ctypes.c_int,
                                                _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int]),
    "ctcdec_decode_batch_host_multi": (ctypes.c_int, [ctypes.POINTER(Config), _vp, _vp, ctypes.c_int, ctypes.c_int,
                                                      _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int]),
    "ctcdec_scorer_create": (ctypes.c_int, [_vp, ctypes.c_double, ctypes.c_double, ctypes.POINTER(ctypes.c_char_p),
                                            ctypes.c_int, ctypes.POINTER(ctypes.c_char_p), ctypes.c_int, ctypes.c_int,
                                            ctypes.c_int, ctypes.POINTER(_vp)]),
    "ctcdec_scorer_create_arpa": (ctypes.c_int, [ctypes.c_char_p, ctypes.c_double, ctypes.c_double,
                                                 ctypes.POINTER(ctypes.c_char_p), ctypes.c_int, ctypes.POINTER(_vp)]),
    "ctcdec_scorer_cond_log_prob": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.POINTER(ctypes.c_double)]),
    "ctcdec_scorer_sent_log_prob": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.POINTER(ctypes.c_double)]),
    "ctcdec_scorer_destroy": (ctypes.c_int, [_vp]),
    "ctcdec_scorer_is_character_based": (ctypes.c_int, [_vp]),
    "ctcdec_scorer_max_order": (ctypes.c_int, [_vp]),
    "ctcdec_scorer_dict_size": (ctypes.c_int, [_vp]),
    "ctcdec_scorer_table_bytes": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_size_t)]),
    "ctcdec_scorer_reset_params": (ctypes.c_int, [_vp, ctypes.c_double, ctypes.c_double]),
    "ctcdec_decode_batch_lm_host": (ctypes.c_int, [ctypes.POINTER(Config), _vp, _vp, _vp, ctypes.c_int, ctypes.c_int,
                                                   _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int]),
    "ctcdec_lm_workspace_bytes": (ctypes.c_int, [ctypes.POINTER(Config), _vp, ctypes.c_int, ctypes.c_int,
                                                 ctypes.POINTER(ctypes.c_size_t)]),
    "ctcdec_decode_batch_lm_device": (ctypes.c_int, [ctypes.POINTER(Config), _vp, _vp, ctypes.c_int, _vp, ctypes.c_int,
                                                     ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                                     ctypes.c_size_t, _vp]),
    "ctcdec_decode_batch_lm_device_async": (ctypes.c_int, [ctypes.POINTER(Config), _vp, _vp, ctypes.c_int, _vp,
                                                           ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp,
                                                           _vp, _vp, ctypes.c_size_t, _vp]),
    "ctcdec_lm_sweep_workspace_bytes": (ctypes.c_int, [ctypes.POINTER(Config), _vp, ctypes.c_int, ctypes.c_int,
                                                       ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]),
    "ctcdec_decode_batch_lm_sweep_async": (ctypes.c_int, [ctypes.POINTER(Config), _vp, _vp, ctypes.c_int, _vp,
                                                          ctypes.c_int, ctypes.c_int, _vp, _vp, ctypes.c_int, _vp, _vp,
                                                          _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_size_t, _vp]),
    "ctcdec_lm_mixed_workspace_bytes": (ctypes.c_int, [ctypes.POINTER(Config), ctypes.POINTER(_vp), ctypes.c_int,
                                                       ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]),
    "ctcdec_decode_batch_lm_mixed_async": (ctypes.c_int, [ctypes.POINTER(Config), ctypes.POINTER(_vp), ctypes.c_int,
                                                          _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, _vp,
                                                          _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_size_t, _vp]),
    "ctcdec_scorer_rescore_rows": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                  ctypes.c_int]),
    "ctcdec_state_create":(ctypes.c_int, [ctypes.POINTER(Config), ctypes.c_int, ctypes.POINTER(_vp)]),
    "ctcdec_state_create_lm": (ctypes.c_int, [ctypes.POINTER(Config), _vp, ctypes.c_int, ctypes.POINTER(_vp)]),
    "ctcdec_state_destroy": (ctypes.c_int, [_vp]),
    "ctcdec_state_frames": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_int)]),
    "ctcdec_decode_stream_host": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp), _vp,
                                                 _vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp]),
    "ctcdec_stream_states_workspace_bytes": (ctypes.c_int, [ctypes.POINTER(_vp), ctypes.c_int, ctypes.c_int,
                                                            ctypes.POINTER(ctypes.c_size_t)]),
    "ctcdec_stream_workspace_bytes": (ctypes.c_int, [ctypes.POINTER(Config), ctypes.c_int, ctypes.c_int,
                                                     ctypes.POINTER(ctypes.c_size_t)]),
    "ctcdec_decode_stream_device": (ctypes.c_int, [_vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int,
                                                   ctypes.POINTER(_vp), _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _vp,
                                                   _vp, _vp, ctypes.c_size_t, _vp]),
    "ctcdec_stream_committed_device": (ctypes.c_int, [ctypes.POINTER(_vp), ctypes.c_int, _vp, _vp, _vp, _vp,
                                                      ctypes.c_int, _vp]),
    "ctcdec_stream_compact": (ctypes.c_int, [ctypes.POINTER(_vp), ctypes.c_int, _vp, _vp]),
    "ctcdec_state_device_bytes": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_size_t)]),
    "ctcdec_profile_enable": (ctypes.c_int, [ctypes.c_int]),
    "ctcdec_profile_read": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float)]),
    "ctcdec_profile_region_cycles": (ctypes.c_int, [_vp]),
    "ctcdec_selftest_math": (ctypes.c_int, [ctypes.c_int, _vp, _vp, _vp, ctypes.c_size_t, ctypes.c_int]),
    "ctcdec_rows_to_host": (ctypes.c_int, [_vp, _vp, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]),
    "ctcdec_selftest_math_f64": (ctypes.c_int, [ctypes.c_int, _vp, _vp, _vp, ctypes.c_size_t, ctypes.c_int]),
}
EXPORTS = tuple(_SIGNATURES)

_lib = None


def load():
    """Loads the CUDA library; raises NativeError if it has not been built (python -m ctcdecode_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(
            "ctcdecode_b200: %s is missing -- build it with `python -m ctcdecode_b200.build` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        if os.environ.get("CTCDECODE_B200_LIB") and not hasattr(lib, name):
            continue  # (an older build of the ABI, loaded for an A/B measurement)
        fn = getattr(lib, name)  # AttributeError here = header / library out of sync
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != OK:
        raise NativeError("ctcdecode_b200 error %d: %s" % (rc, load().ctcdec_last_error().decode()))
