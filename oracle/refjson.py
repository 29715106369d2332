"""ctypes binding of oracle/_ref/libblah2json.so: the reference's UNMODIFIED Map::to_json + Map::delay_bin_to_km and
rapidjson's write / read / write of single doubles (oracle/json/ref_json_capi.cpp).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libblah2json.so")
_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise FileNotFoundError(f"{LIB_PATH} missing: run `make -C oracle/json REF=<blah2 checkout>`")
        _lib = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)
        _lib.refjson_format_doubles.restype = C.c_int64
        _lib.refjson_format_doubles.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
        _lib.refjson_map_json.restype = C.c_int64
        _lib.refjson_map_json.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_double,
                                          C.c_double, C.c_uint64, C.c_uint32, C.c_void_p, C.c_size_t]
    return _lib


def format_doubles_bytes(values) -> bytes:
    """The comma-separated texts of the values (an empty field where a value has none)."""
    v = np.ascontiguousarray(np.asarray(values, dtype=np.float64).ravel())
    out = np.empty(v.size * 25 + 1, dtype=np.uint8)
    n = lib().refjson_format_doubles(v.ctypes.data, v.size, out.ctypes.data, out.size)
    assert 0 <= n <= out.size
    return out[:n].tobytes()


def format_doubles(values) -> list[str]:
    return format_doubles_bytes(values).decode("ascii").split(",")


def map_json(m, delay, doppler, noise, maxp, ts, fs) -> bytes:
    """delay_bin_to_km(to_json(ts), fs) of a Map holding m [nDop, nDel] complex, the axes and the metrics."""
    m = np.ascontiguousarray(m, dtype=np.complex128)
    delay = np.ascontiguousarray(delay, dtype=np.int32)
    doppler = np.ascontiguousarray(doppler, dtype=np.float64)
    cap = m.size * 27 + 64 * (delay.size + doppler.size) + 1024
    out = np.empty(cap, dtype=np.uint8)
    n = lib().refjson_map_json(m.ctypes.data, m.shape[0], m.shape[1], delay.ctypes.data, doppler.ctypes.data,
                               float(noise), float(maxp), int(ts), int(fs), out.ctypes.data, cap)
    assert 0 < n <= cap
    return out[:n].tobytes()
