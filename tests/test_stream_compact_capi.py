"""Argument checks of the streaming compaction entry points (no GPU needed): ctcdec_stream_compact and
ctcdec_state_device_bytes reject bad arguments before they read a state or touch a device.  (Refusals that need real
states -- hook scorers, graph capture -- are in tests/test_gpu_stream_compact.py.)"""
import ctypes

import pytest

from ctcdecode_b200 import _native, build as libbuild


@pytest.fixture(scope="module")
def lib():
    libbuild.build()
    return _native.load()


def test_stream_compact_arguments(lib):
    kept = (ctypes.c_int64 * 2)()
    assert lib.ctcdec_stream_compact(None, 0, None, None) == 0                  # nothing to do
    assert lib.ctcdec_stream_compact(None, -1, kept, None) == -1
    assert b"negative" in lib.ctcdec_last_error()
    assert lib.ctcdec_stream_compact(None, 2, kept, None) == -1                 # states NULL
    assert b"NULL" in lib.ctcdec_last_error()
    nulls = (ctypes.c_void_p * 2)(None, None)
    assert lib.ctcdec_stream_compact(nulls, 2, kept, None) == -1
    assert b"states[0] is NULL" in lib.ctcdec_last_error()
    # the same object twice is refused before either is read (the pointer need not be a state)
    buf = ctypes.create_string_buffer(64)
    dup = (ctypes.c_void_p * 3)(ctypes.addressof(buf), None, ctypes.addressof(buf))
    assert lib.ctcdec_stream_compact(dup, 3, kept, None) == -1
    assert b"states[1] is NULL" in lib.ctcdec_last_error()
    dup = (ctypes.c_void_p * 2)(ctypes.addressof(buf), ctypes.addressof(buf))
    assert lib.ctcdec_stream_compact(dup, 2, kept, None) == -1
    assert b"same object" in lib.ctcdec_last_error()


def test_state_device_bytes_arguments(lib):
    n = ctypes.c_size_t(0)
    assert lib.ctcdec_state_device_bytes(None, ctypes.byref(n)) == -1
    buf = ctypes.create_string_buffer(64)
    assert lib.ctcdec_state_device_bytes(ctypes.addressof(buf), None) == -1
    assert b"NULL" in lib.ctcdec_last_error()


@pytest.mark.parametrize("name", ["ctcdec_stream_compact", "ctcdec_state_device_bytes"])
def test_exported(lib, name):
    assert name in _native.EXPORTS and hasattr(lib, name)
