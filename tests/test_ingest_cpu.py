"""CPU: the int8 (HackRF, Kraken) and complex float32 (USRP) host entry points refuse null arguments before any device
call, and the numpy statement of the samples blah2 takes from those sources holds on hand-built values."""
import ctypes as C

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import Pipeline
from blah2_b200.scene import iq_from_cf32, iq_from_ci8


def test_null_arguments_are_refused_without_a_device():
    lib = capi.load()
    x8 = np.zeros(8, dtype=np.int8)
    xf = np.zeros(8, dtype=np.float32)
    m = np.zeros(4, dtype=np.complex128)
    for name, buf in (("b200dd_pipeline_submit_host_ci8", x8), ("b200dd_pipeline_submit_host_cf32", xf)):
        fn = getattr(lib, name)
        assert fn(None, capi.ptr(buf), capi.ptr(buf), 4, capi.ptr(m)) == capi.ERR_ARG
        assert name.encode() in lib.b200dd_last_error() and b"null" in lib.b200dd_last_error()
        assert fn(None, None, capi.ptr(buf), 4, None) == capi.ERR_ARG
        assert fn(None, capi.ptr(buf), None, 4, None) == capi.ERR_ARG
        assert fn(None, None, None, 0, None) == capi.ERR_ARG


def test_ci8_bytes_are_read_as_int8():
    """HackRf.cpp:116-128 and Kraken.cpp:97-112: `{(double)buf[i], (double)buf[i+1]}` with buf an int8_t pointer, so
    rtl-sdr's offset-binary bytes keep no offset: 0x7F -> 127, 0x80 -> -128, 0xFF -> -1."""
    raw = np.array([0x7F, 0x80, 0xFF, 0x00, 0x01, 0xFE, 0x81, 0x7E], dtype=np.uint8)
    got = iq_from_ci8(raw)
    assert got.dtype == np.complex128
    assert np.array_equal(got.real, [127.0, -1.0, 1.0, -127.0])
    assert np.array_equal(got.imag, [-128.0, 0.0, -2.0, 126.0])
    assert np.array_equal(iq_from_ci8(raw.view(np.int8)), got)  # HackRF's int8 buffer: the same values
    # every byte value, in both positions of a pair
    allb = np.arange(256, dtype=np.uint8)
    pairs = iq_from_ci8(np.stack([allb, allb[::-1]], axis=1).ravel())
    want = np.where(allb < 128, allb.astype(np.float64), allb.astype(np.float64) - 256.0)
    assert np.array_equal(pairs.real, want) and np.array_equal(pairs.imag, want[::-1])


def test_cf32_floats_are_widened_exactly():
    """Usrp.cpp:54-91: `{(double)re, (double)im}` of UHD's fc32 samples -- signed zeros, subnormals and sc16/32768
    values keep their exact value."""
    sub = np.float32(1e-45)  # the smallest float32 subnormal, 2^-149
    vals = np.array([0.0, -0.0, sub, -sub, -32768 / 32768, 32767 / 32768, 12345 / 32768, -1 / 32768,
                     np.float32(0.1), np.float32(-3.4e38)], dtype=np.float32)
    buf = vals.reshape(-1, 2).copy().view(np.complex64).ravel()
    got = iq_from_cf32(buf)
    assert got.dtype == np.complex128 and got.shape == (5,)
    flat = np.stack([got.real, got.imag], axis=1).ravel()
    assert np.array_equal(flat, vals.astype(np.float64))
    assert np.array_equal(np.signbit(flat), np.signbit(vals))  # -0.0 stays -0.0, in either part
    assert flat[2] == 2.0 ** -149 and flat[3] == -(2.0 ** -149)
    assert flat[5] == 32767 / 32768 and flat[6] == 12345 / 32768 and flat[7] == -1 / 32768
    assert flat[8] == float(np.float32(0.1)) and flat[8] != 0.1
    assert np.array_equal(iq_from_cf32(vals), got)  # a float32 buffer of interleaved I, Q: the same samples


def test_python_entries_check_their_buffers_before_the_library():
    """Pipeline.submit_host_ci8 / _cf32 take two contiguous buffers of the format's dtype and equal length; anything
    else is a ValueError before a call into the library (no pipeline is needed to see it)."""
    p = Pipeline.__new__(Pipeline)
    bad = [(p.submit_host_ci8, np.zeros(8, np.int16), np.zeros(8, np.int8)),
           (p.submit_host_ci8, np.zeros(8, np.int8), np.zeros(6, np.int8)),
           (p.submit_host_ci8, np.zeros(7, np.int8), np.zeros(7, np.int8)),
           (p.submit_host_ci8, np.zeros((8, 2), np.int8)[:, 0], np.zeros(8, np.int8)),
           (p.submit_host_cf32, np.zeros(4, np.complex128), np.zeros(4, np.complex64)),
           (p.submit_host_cf32, np.zeros(4, np.complex64), np.zeros(5, np.complex64)),
           (p.submit_host_cf32, np.zeros(8, np.float32), np.zeros(8, np.float32))]
    for f, x, y in bad:
        with pytest.raises(ValueError):
            f(x, y)
