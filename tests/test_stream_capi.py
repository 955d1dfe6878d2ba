"""Argument checks of the device streaming entry points (no GPU needed): ctcdec_stream_workspace_bytes,
ctcdec_decode_stream_device and ctcdec_stream_committed_device reject bad arguments before touching a device.
(States from different configurations and scorer states need real states: tests/test_gpu_stream_device.py.)"""
import ctypes

import pytest

from ctcdecode_b200 import _native, build as libbuild


@pytest.fixture(scope="module")
def lib():
    libbuild.build()
    return _native.load()


def test_stream_workspace_bytes(lib):
    cfg = _native.Config(29, 100, 0, 0, 40, 1.0)
    n = ctypes.c_size_t(0)
    assert lib.ctcdec_stream_workspace_bytes(ctypes.byref(cfg), 256, 16, ctypes.byref(n)) == 0
    # the pruned rows of the chunk (256 x 16 x 32 floats) and the per-stream tables, no arena
    assert 256 * 16 * 32 * 4 < n.value < 256 * 16 * 32 * 4 + 256 * 64 + 4096
    m = ctypes.c_size_t(0)
    assert lib.ctcdec_stream_workspace_bytes(ctypes.byref(cfg), 256, 32, ctypes.byref(m)) == 0 and m.value > n.value
    assert lib.ctcdec_stream_workspace_bytes(ctypes.byref(cfg), 256, 16, None) == -1
    bad = _native.Config(29, 0, 0, 0, 40, 1.0)
    assert lib.ctcdec_stream_workspace_bytes(ctypes.byref(bad), 1, 16, ctypes.byref(n)) == -2


def _dev(lib, B, states, dtype=-1, eos=None):
    eos = eos if eos is not None else (ctypes.c_uint8 * max(B, 1))()
    return lib.ctcdec_decode_stream_device(None, dtype, None, B, 4, states, eos, None, None, 0, None, None, None, None,
                                           None, 0, None)


def test_decode_stream_device_arguments(lib):
    assert _dev(lib, 0, None) == 0                      # nothing to do
    assert _dev(lib, -1, None) == -1
    assert _dev(lib, 1, None, dtype=7) == -1            # dtype checked first
    assert b"dtype" in lib.ctcdec_last_error()
    assert _dev(lib, 1, None) == -1                     # states NULL
    assert b"NULL" in lib.ctcdec_last_error()
    nulls = (ctypes.c_void_p * 2)(None, None)
    assert _dev(lib, 2, nulls) == -1
    assert b"states[0] is NULL" in lib.ctcdec_last_error()
    assert lib.ctcdec_decode_stream_device(None, -1, None, 2, 4, nulls, None, None, None, 0, None, None, None, None,
                                           None, 0, None) == -1  # is_eos NULL


def test_stream_committed_device_arguments(lib):
    c = (ctypes.c_int32 * 2)()
    nulls = (ctypes.c_void_p * 2)(None, None)
    assert lib.ctcdec_stream_committed_device(None, 0, None, None, None, None, 0, None) == 0
    assert lib.ctcdec_stream_committed_device(None, -3, None, c, None, None, 0, None) == -1
    assert lib.ctcdec_stream_committed_device(nulls, 2, None, None, None, None, 0, None) == -1  # committed NULL
    assert lib.ctcdec_stream_committed_device(nulls, 2, None, c, None, None, -1, None) == -1   # cap < 0
    assert lib.ctcdec_stream_committed_device(nulls, 2, None, c, None, None, 8, None) == -1    # cap > 0, no rows
    assert b"tokens" in lib.ctcdec_last_error()
    assert lib.ctcdec_stream_committed_device(None, 2, None, c, None, None, 0, None) == -1     # states NULL
    assert lib.ctcdec_stream_committed_device(nulls, 2, None, c, None, None, 0, None) == -1
    assert b"states[0] is NULL" in lib.ctcdec_last_error()
