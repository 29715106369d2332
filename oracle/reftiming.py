"""ctypes binding of oracle/_ref/libblah2timing.so: the reference's UNMODIFIED Timing::update / Timing::to_json
(oracle/timing/ref_timing_capi.cpp).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libblah2timing.so")
_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise FileNotFoundError(f"{LIB_PATH} missing: run `make -C oracle/timing REF=<blah2 checkout>`")
        _lib = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)
        _lib.reftiming_json.restype = C.c_int64
        _lib.reftiming_json.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_char_p), C.c_void_p,
                                        C.c_uint32, C.c_void_p, C.c_size_t]
    return _lib


def timing_json(t_start, t_now, n, names, values) -> bytes:
    """Timing(t_start), then the n-th update(t_now, values, names), then to_json()."""
    v = np.ascontiguousarray(np.asarray(values, dtype=np.float64).ravel())
    arr = (C.c_char_p * max(v.size, 1))(*[s.encode() for s in names])
    cap = 4096
    out = np.empty(cap, dtype=np.uint8)
    k = lib().reftiming_json(int(t_start), int(t_now), int(n), arr, v.ctypes.data, v.size, out.ctypes.data, cap)
    assert 0 < k <= cap
    return out[:k].tobytes()
