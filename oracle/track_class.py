"""ctypes binding of the Tracker / Track class harness (oracle/trackclass/track_class_capi.cpp), built with the
reference's own classes (oracle/_ref/libtrackclass_ref.so) and with the drop-in classes
(oracle/_ref/libtrackclass_dropin.so).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIBS = {"ref": os.path.join(_HERE, "_ref", "libtrackclass_ref.so"),
        "dropin": os.path.join(_HERE, "_ref", "libtrackclass_dropin.so")}
C_LIGHT = 299792458  # Constants::c, a uint32_t
_libs = {}


def available(which) -> bool:
    return os.path.exists(LIBS[which])


def lib(which):
    if which not in _libs:
        if not available(which):
            raise FileNotFoundError(f"{LIBS[which]} missing: run build()")
        L = C.CDLL(LIBS[which], mode=os.RTLD_LOCAL)
        i64, vp = C.c_int64, C.c_void_p
        for name, res, args in [
            ("tc_last_error", C.c_char_p, []),
            ("tc_create", vp, [C.c_uint32, C.c_uint32, C.c_uint32] + [C.c_double] * 4),
            ("tc_destroy", None, [vp]),
            ("tc_process", i64, [vp, vp, vp, vp, C.c_uint32, C.c_uint64, C.POINTER(i64)]),
            ("tc_keep", i64, [vp]),
            ("tc_to_json", i64, [vp, i64, C.c_uint64, vp, C.c_size_t, C.POINTER(i64)]),
            ("tc_save", i64, [vp, i64, C.c_uint64, C.c_char_p]),
            ("tc_get_n", i64, [vp, i64]),
            ("tc_get_nstate", i64, [vp, i64, C.c_char_p]),
            ("tc_predict", i64, [vp] + [C.c_double] * 4 + [vp]),
        ]:
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _libs[which] = L
    return _libs[which]


class ClassError(RuntimeError):
    pass


class TrackerClass:
    """`Tracker tracker(m, n, nDelete, cpi, maxAcc, rangeRes, lambda)` of one build, with rangeRes = c / fs and
    lambda = c / fc as blah2.cpp:193-194 computes them (or given directly as range_res / lam)."""

    def __init__(self, which, m, n, nDelete, cpi, maxAcc, fs=None, fc=None, range_res=None, lam=None):
        self._lib = lib(which)
        rr = float(C_LIGHT) / int(fs) if range_res is None else float(range_res)
        la = float(C_LIGHT) / int(fc) if lam is None else float(lam)
        self._h = self._lib.tc_create(int(m), int(n), int(nDelete), float(cpi), float(maxAcc), rr, la)
        if not self._h:
            raise ClassError(self._lib.tc_last_error().decode())
        self._out = np.empty(1 << 16, dtype=np.uint8)
        self.ns_process = self.ns_json = 0

    def _check(self, v):
        if v < 0:
            raise ClassError(self._lib.tc_last_error().decode())
        return v

    def process(self, delay, doppler, snr, ts):
        """track = tracker.process(&detection, ts)"""
        v = [np.ascontiguousarray(np.asarray(a, dtype=np.float64).ravel()) for a in (delay, doppler, snr)]
        assert v[0].size == v[1].size == v[2].size
        ns = C.c_int64()
        self._check(self._lib.tc_process(self._h, v[0].ctypes.data, v[1].ctypes.data, v[2].ctypes.data, v[0].size,
                                         int(ts), C.byref(ns)))
        self.ns_process = ns.value

    def keep(self) -> int:
        """Index of a kept copy of the last track."""
        return self._lib.tc_keep(self._h)

    def to_json(self, ts, k=-1) -> bytes:
        ns = C.c_int64()
        while True:
            n = self._check(self._lib.tc_to_json(self._h, int(k), int(ts), self._out.ctypes.data, self._out.size,
                                                 C.byref(ns)))
            if n <= self._out.size:
                self.ns_json = ns.value
                return self._out[:n].tobytes()
            self._out = np.empty(2 * n, dtype=np.uint8)

    def save(self, ts, path, k=-1) -> bool:
        return bool(self._check(self._lib.tc_save(self._h, int(k), int(ts), os.fsencode(path))))

    def get_n(self, k=-1) -> int:
        return self._check(self._lib.tc_get_n(self._h, int(k)))

    def get_nState(self, state, k=-1) -> int:
        return self._check(self._lib.tc_get_nstate(self._h, int(k), state.encode()))

    def predict(self, delay, doppler, acc, T):
        out = np.empty(2, dtype=np.float64)
        self._check(self._lib.tc_predict(self._h, float(delay), float(doppler), float(acc), float(T),
                                         out.ctypes.data))
        return float(out[0]), float(out[1])

    def close(self):
        if self._h:
            self._lib.tc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
