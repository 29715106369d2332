"""ctypes binding of oracle/_ref/libblah2detjson.so: the reference's UNMODIFIED Detection::to_json +
Detection::delay_bin_to_km (oracle/detjson/ref_detjson_capi.cpp).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libblah2detjson.so")
_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise FileNotFoundError(f"{LIB_PATH} missing: run `make -C oracle/detjson REF=<blah2 checkout>`")
        _lib = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)
        _lib.refdetjson_detection_json.restype = C.c_int64
        _lib.refdetjson_detection_json.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64,
                                                   C.c_uint32, C.c_void_p, C.c_size_t]
    return _lib


def detection_json(delay, doppler, snr, ts, fs) -> bytes:
    """delay_bin_to_km(to_json(ts), fs) of a Detection holding the three lists (delay in bins)."""
    v = [np.ascontiguousarray(np.asarray(a, dtype=np.float64).ravel()) for a in (delay, doppler, snr)]
    assert v[0].size == v[1].size == v[2].size
    cap = 75 * v[0].size + 128
    out = np.empty(cap, dtype=np.uint8)
    n = lib().refdetjson_detection_json(v[0].ctypes.data, v[1].ctypes.data, v[2].ctypes.data, v[0].size, int(ts),
                                        int(fs), out.ctypes.data, cap)
    assert 0 < n <= cap
    return out[:n].tobytes()
