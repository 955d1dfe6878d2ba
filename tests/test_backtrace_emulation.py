"""CPU tests of the backtrace in the beam program's epilogue (BeamParams::backtrace, beam_program.cuh): an offline
decode of an uncut vocabulary runs finalize_cta_run inside the beam CTA, with the CTA's own threads, in the shared
memory behind the layout's head.  Through the emulation (tests/native/emulate_backtrace.cpp) the results must equal
those of the separate finalize pass (tests/emul.py) bit for bit, at every block size and emulated thread order, and
match the oracle."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from ctcdecode_b200.synth import ctc_like_probs, flat_probs
from tests import emul
from tests.parity import compare

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "native", "emulate_backtrace.cpp")
_OUT = os.path.join(_HERE, "native", "_build", "libctc_emul_backtrace.so")
_i32p = ctypes.POINTER(ctypes.c_int32)
_f32p = ctypes.POINTER(ctypes.c_float)
_lib = None


def _build():
    """Compiles tests/native/emulate_backtrace.cpp (which includes emulate_cta.cpp) like tests/emul.py does."""
    global _lib
    if _lib is None:
        os.makedirs(os.path.dirname(_OUT), exist_ok=True)
        csrc = os.path.join(_HERE, "..", "ctcdecode_b200", "csrc")
        deps = [_SRC, os.path.join(_HERE, "native", "emulate_cta.cpp")] + \
            [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not (os.path.exists(_OUT) and all(os.path.getmtime(_OUT) >= os.path.getmtime(d) for d in deps)):
            tmp = _OUT + ".tmp%d" % os.getpid()
            subprocess.run(["g++", "-O2", "-std=c++17", "-mfma", "-ffp-contract=off", "-fPIC", "-shared",
                            "-nostdlib++", "-Wno-unused-function", "-pthread", _SRC, "-o", tmp, "-l:libstdc++.so.6",
                            "-lm"], check=True)
            os.replace(tmp, _OUT)
        _lib = ctypes.CDLL(_OUT)
        _lib.emu_decode_batch_backtrace.restype = ctypes.c_int
        _lib.emu_decode_batch_backtrace.argtypes = [_f32p, _i32p] + [ctypes.c_int] * 4 + [ctypes.c_double] + \
            [ctypes.c_int] * 4 + [_i32p, _i32p, _f32p, _i32p, _i32p, _i32p]
    return _lib


def decode_backtrace(probs, seq_lens=None, beam=100, blank_id=0, log_input=False, nt=0):
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    B, T, V = probs.shape
    sl = None if seq_lens is None else np.ascontiguousarray(seq_lens, dtype=np.int32)
    out = dict(tokens=np.full((B, beam, T), -1, np.int32), timesteps=np.full((B, beam, T), -1, np.int32),
               scores=np.zeros((B, beam), np.float32), lens=np.zeros((B, beam), np.int32),
               n_results=np.zeros((B,), np.int32), ties=np.zeros((B,), np.int32))
    rc = _build().emu_decode_batch_backtrace(
        probs.ctypes.data_as(_f32p), sl.ctypes.data_as(_i32p) if sl is not None else None, B, T, V, beam, 1.0, V,
        blank_id, int(log_input), nt, out["tokens"].ctypes.data_as(_i32p), out["timesteps"].ctypes.data_as(_i32p),
        out["scores"].ctypes.data_as(_f32p), out["lens"].ctypes.data_as(_i32p),
        out["n_results"].ctypes.data_as(_i32p), out["ties"].ctypes.data_as(_i32p))
    assert rc == 0, rc
    return out


def _same_as_finalize_pass(probs, seq_lens=None, **kw):
    got = decode_backtrace(probs, seq_lens, **kw)
    V = probs.shape[2]
    ref = emul.decode(probs, seq_lens, cutoff_prob=1.0, cutoff_top_n=V, **kw)
    for k in ref:
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    return got


@pytest.mark.parametrize("nt", [128, 160, 192, 256, 512, 1024])
@pytest.mark.parametrize("beam", [16, 40, 100, 200])
def test_backtrace_in_epilogue_any_block_size(nt, beam):
    probs = ctc_like_probs(2, 120, 29, seed=60).numpy()
    _same_as_finalize_pass(probs, beam=beam, nt=nt)


@pytest.mark.parametrize("order", [1, 2, 3, 7])
def test_backtrace_in_epilogue_emulated_thread_order(monkeypatch, order):
    """The program's result must not depend on the order the emulation runs its threads in."""
    monkeypatch.setenv("CTC_EMU_ORDER", str(order))
    probs = ctc_like_probs(3, 150, 29, seed=61).numpy()
    _same_as_finalize_pass(probs, beam=100)
    _same_as_finalize_pass(probs, beam=100, nt=128)


def test_backtrace_in_epilogue_ragged_empty_and_log_input():
    probs = ctc_like_probs(6, 60, 29, seed=62).numpy()
    _same_as_finalize_pass(probs, np.array([60, 0, 1, 17, 59, 1000], np.int32), beam=16)
    _same_as_finalize_pass(probs[:, :0], beam=16)
    logp = ctc_like_probs(3, 80, 29, seed=63, log=True).numpy()
    _same_as_finalize_pass(logp, beam=32, log_input=True)


def test_backtrace_in_epilogue_beam_not_full_and_flat_rows():
    _same_as_finalize_pass(flat_probs(2, 6, 3, 64).numpy(), beam=64)
    _same_as_finalize_pass(flat_probs(2, 200, 5, 65, temp=2.0).numpy(), beam=16)


def test_backtrace_in_epilogue_matches_oracle(cport):
    probs = ctc_like_probs(4, 300, 29, seed=66).numpy()
    got = decode_backtrace(probs, beam=100)
    ref = cport.decode_alternatives(probs, None, beam=100, cutoff_top_n=29)
    checked, _ = compare(ref, got, ref["ties"], "backtrace-epilogue")
    assert checked > 0
    assert np.array_equal(ref["ties"] != 0, (got["ties"] & 7) != 0)


def test_cut_vocabulary_keeps_the_finalize_pass():
    probs = ctc_like_probs(1, 20, 29, seed=67).numpy()
    f = _build().emu_decode_batch_backtrace
    B, T, V = probs.shape
    z = np.zeros((B, 16, T), np.int32)
    rc = f(probs.ctypes.data_as(_f32p), None, B, T, V, 16, 1.0, 10, 0, 0, 0, z.ctypes.data_as(_i32p),
           z.ctypes.data_as(_i32p), np.zeros((B, 16), np.float32).ctypes.data_as(_f32p),
           np.zeros((B, 16), np.int32).ctypes.data_as(_i32p), np.zeros(B, np.int32).ctypes.data_as(_i32p),
           np.zeros(B, np.int32).ctypes.data_as(_i32p))
    assert rc != 0
