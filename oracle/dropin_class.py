"""ctypes binding of the class harness oracle/dropinclass/class_capi.cpp, built with the reference's own classes
(oracle/_ref/libdropinclass_ref.so) and with the drop-in classes (oracle/_ref/libdropinclass_dropin.so).  Every
object is created once and called many times, as blah2.cpp calls its objects once per CPI.  TEST INFRASTRUCTURE
ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIBS = {"ref": os.path.join(_HERE, "_ref", "libdropinclass_ref.so"),
        "dropin": os.path.join(_HERE, "_ref", "libdropinclass_dropin.so")}
_libs = {}


def available(which) -> bool:
    return os.path.exists(LIBS[which])


def lib(which):
    if which not in _libs:
        if not available(which):
            raise FileNotFoundError(f"{LIBS[which]} missing: run build()")
        L = C.CDLL(LIBS[which], mode=os.RTLD_LOCAL)
        i64, u32, d, vp, i = C.c_int64, C.c_uint32, C.c_double, C.c_void_p, C.c_int
        for name, res, args in [
            ("dc_last_error", C.c_char_p, []),
            ("dc_spectrum_create", vp, [u32, d]),
            ("dc_spectrum_destroy", None, [vp]),
            ("dc_spectrum_process", i64, [vp, vp, u32, vp, vp, u32, vp]),
            ("dc_cfar_create", vp, [d, i, i, i, d]),
            ("dc_cfar_destroy", None, [vp]),
            ("dc_cfar_process", i64, [vp, vp, u32, u32, vp, vp, d, vp, vp, vp, u32]),
            ("dc_centroid_create", vp, [u32, u32, d]),
            ("dc_centroid_destroy", None, [vp]),
            ("dc_centroid_process", i64, [vp, vp, vp, vp, u32, vp, vp, vp, u32]),
            ("dc_interpolate_create", vp, [i, i]),
            ("dc_interpolate_destroy", None, [vp]),
            ("dc_interpolate_process", i64, [vp, vp, vp, vp, u32, vp, u32, u32, vp, vp, d, vp, vp, vp, u32]),
            ("dc_pair_create", vp, [C.c_int32] * 4 + [u32, u32, i, i, C.c_int32, C.c_int32, u32]),
            ("dc_pair_destroy", None, [vp]),
            ("dc_pair_push", None, [vp, vp, u32, vp, u32]),
            ("dc_pair_filter", i64, [vp]),
            ("dc_pair_ambiguity", i64, [vp, vp]),
            ("dc_pair_n_samples", u32, [vp]),
            ("dc_pair_fifo", u32, [vp, i, vp, u32]),
        ]:
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _libs[which] = L
    return _libs[which]


class ClassError(RuntimeError):
    pass


def _c128(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.complex128).ravel())


def _f64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64).ravel())


class _Object:
    _kind = ""

    def __init__(self, which, *args):
        self._lib = lib(which)
        self._h = getattr(self._lib, f"dc_{self._kind}_create")(*args)
        if not self._h:
            raise ClassError(self._lib.dc_last_error().decode())

    def _check(self, v):
        if v < 0:
            raise ClassError(self._lib.dc_last_error().decode())
        return v

    def _list(self, fn, *args, cap):
        out = [np.empty(max(1, cap), dtype=np.float64) for _ in range(3)]
        n = self._check(fn(self._h, *args, *[o.ctypes.data for o in out], max(1, cap)))
        assert n <= max(1, cap)
        return tuple(o[:n].copy() for o in out)

    def close(self):
        if self._h:
            getattr(self._lib, f"dc_{self._kind}_destroy")(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SpectrumAnalyserClass(_Object):
    """`SpectrumAnalyser(n, bandwidth)`; process(x) runs it on a new FIFO holding x."""
    _kind = "spectrum"

    def process(self, x):
        """(spectrum, frequency, samples left in the FIFO)"""
        x = _c128(x)
        cap = 1 << 17
        spec = np.empty(cap, dtype=np.complex128)
        freq = np.empty(cap, dtype=np.float64)
        counts = np.zeros(3, dtype=np.uint32)
        self._check(self._lib.dc_spectrum_process(self._h, x.ctypes.data, x.size, spec.ctypes.data, freq.ctypes.data,
                                                  cap, counts.ctypes.data))
        assert counts[0] <= cap and counts[1] <= cap
        return spec[:counts[0]].copy(), freq[:counts[1]].copy(), int(counts[2])


def _map_args(m, delay, doppler):
    m = _c128(np.asarray(m).reshape(-1))
    return m, np.ascontiguousarray(delay, dtype=np.int32), _f64(doppler)


class CfarClass(_Object):
    """`CfarDetector1D(pfa, nGuard, nTrain, minDelay, minDoppler)` (the int8_t parameters narrowed as C++ does)."""
    _kind = "cfar"

    def process(self, m, delay, doppler, noisePower):
        shape = np.shape(m)
        mm, dl, dp = _map_args(m, delay, doppler)
        return self._list(self._lib.dc_cfar_process, mm.ctypes.data, shape[0], shape[1], dl.ctypes.data,
                          dp.ctypes.data, float(noisePower), cap=mm.size)


class CentroidClass(_Object):
    """`Centroid(nDelay, nDoppler, resolutionDoppler)`"""
    _kind = "centroid"

    def process(self, delay, doppler, snr):
        d, f, s = _f64(delay), _f64(doppler), _f64(snr)
        return self._list(self._lib.dc_centroid_process, d.ctypes.data, f.ctypes.data, s.ctypes.data, d.size,
                          cap=d.size)


class InterpolateClass(_Object):
    """`Interpolate(doDelay, doDoppler)`"""
    _kind = "interpolate"

    def process(self, delay, doppler, snr, m, mdelay, mdoppler, noisePower):
        d, f, s = _f64(delay), _f64(doppler), _f64(snr)
        shape = np.shape(m)
        mm, dl, dp = _map_args(m, mdelay, mdoppler)
        return self._list(self._lib.dc_interpolate_process, d.ctypes.data, f.ctypes.data, s.ctypes.data, d.size,
                          mm.ctypes.data, shape[0], shape[1], dl.ctypes.data, dp.ctypes.data, float(noisePower),
                          cap=d.size)


class PairClass(_Object):
    """Two FIFOs of capacity fifo_cap with `Ambiguity(delayMin, delayMax, dopplerMin, dopplerMax, fs, n,
    roundHamming)` and, where clutter is (delayMin, delayMax), `WienerHopf(delayMin, delayMax, n)` reading them."""
    _kind = "pair"

    def __init__(self, which, delayMin, delayMax, dopplerMin, dopplerMax, fs, n, roundHamming, clutter, fifo_cap):
        cl = clutter if clutter is not None else (0, 0)
        super().__init__(which, delayMin, delayMax, dopplerMin, dopplerMax, fs, n, int(roundHamming),
                         int(clutter is not None), cl[0], cl[1], fifo_cap)
        self.fifo_cap = fifo_cap

    def push(self, x, y):
        x, y = _c128(x), _c128(y)
        self._lib.dc_pair_push(self._h, x.ctypes.data, x.size, y.ctypes.data, y.size)

    def filter(self) -> bool:
        return bool(self._check(self._lib.dc_pair_filter(self._h)))

    def ambiguity(self, shape):
        m = np.empty(shape, dtype=np.complex128)
        self._check(self._lib.dc_pair_ambiguity(self._h, m.ctypes.data))
        return m

    def n_samples(self) -> int:
        return int(self._lib.dc_pair_n_samples(self._h))

    def fifo(self, which):
        """Every sample queued in x (0) or y (1), front first."""
        out = np.empty(self.fifo_cap, dtype=np.complex128)
        n = self._lib.dc_pair_fifo(self._h, int(which), out.ctypes.data, self.fifo_cap)
        assert n <= self.fifo_cap
        return out[:n].copy()
