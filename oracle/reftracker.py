"""ctypes binding of oracle/_ref/libblah2tracker.so: the reference's UNMODIFIED Tracker::process + Track::to_json
(oracle/tracker/ref_tracker_capi.cpp).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libblah2tracker.so")
C_LIGHT = 299792458  # Constants::c, a uint32_t
_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise FileNotFoundError(f"{LIB_PATH} missing: run `make -C oracle/tracker REF=<blah2 checkout>`")
        _lib = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)
        _lib.reftracker_create.restype = C.c_void_p
        _lib.reftracker_create.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, C.c_double, C.c_double,
                                           C.c_double]
        _lib.reftracker_destroy.restype = None
        _lib.reftracker_destroy.argtypes = [C.c_void_p]
        _lib.reftracker_process.restype = C.c_int64
        _lib.reftracker_process.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64,
                                            C.c_void_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        _lib.reftracker_copy.restype = C.c_int64
        _lib.reftracker_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    return _lib


class RefTracker:
    """Tracker(m, n, nDelete, cpi, maxAcc, c / fs, c / fc) as blah2.cpp:186-195 constructs it."""

    def __init__(self, m, n, nDelete, cpi, maxAcc, fs, fc):
        self._h = lib().reftracker_create(int(m), int(n), int(nDelete), float(cpi), float(maxAcc),
                                          float(C_LIGHT) / int(fs), float(C_LIGHT) / int(fc))
        assert self._h
        self._out = np.empty(1 << 16, dtype=np.uint8)
        self.ns_process = self.ns_json = 0

    def process(self, delay, doppler, snr, ts) -> bytes:
        """tracker->process(detection, ts)->to_json(ts): the document (truncated where the Writer stopped)."""
        v = [np.ascontiguousarray(np.asarray(a, dtype=np.float64).ravel()) for a in (delay, doppler, snr)]
        assert v[0].size == v[1].size == v[2].size
        tp, tj = C.c_int64(), C.c_int64()
        n = lib().reftracker_process(self._h, v[0].ctypes.data, v[1].ctypes.data, v[2].ctypes.data, v[0].size,
                                     int(ts), self._out.ctypes.data, self._out.size, C.byref(tp), C.byref(tj))
        assert n >= 0
        self.ns_process, self.ns_json = tp.value, tj.value
        if n > self._out.size:
            self._out = np.empty(2 * n, dtype=np.uint8)
            lib().reftracker_copy(self._h, self._out.ctypes.data, self._out.size)
        return self._out[:n].tobytes()

    def close(self):
        if self._h:
            lib().reftracker_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
