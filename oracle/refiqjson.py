"""ctypes binding of oracle/_ref/libblah2iqjson.so: the reference's UNMODIFIED IqData::to_json
(oracle/iqjson/ref_iqjson_capi.cpp).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libblah2iqjson.so")
_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise FileNotFoundError(f"{LIB_PATH} missing: run `make -C oracle/iqjson REF=<blah2 checkout>`")
        _lib = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)
        _lib.refiqjson_iqdata_json.restype = C.c_int64
        _lib.refiqjson_iqdata_json.argtypes = [C.c_void_p, C.c_uint32, C.c_double, C.c_double, C.c_double,
                                               C.c_uint64, C.c_void_p, C.c_size_t]
    return _lib


def iqdata_json(spectrum, mn, mx, mean, ts) -> bytes:
    """IqData::to_json(ts) of an IqData holding the complex bins and the metrics min, max, mean; the truncated text
    where rapidjson's Writer stops at a bin without JSON text."""
    s = np.ascontiguousarray(np.asarray(spectrum, dtype=np.complex128).ravel())
    cap = 32 * s.size + 256
    out = np.empty(cap, dtype=np.uint8)
    n = lib().refiqjson_iqdata_json(s.ctypes.data, s.size, float(mn), float(mx), float(mean), int(ts), out.ctypes.data,
                                    cap)
    assert 0 < n <= cap
    return out[:n].tobytes()
