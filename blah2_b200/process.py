"""Host-side mirror of the reference's process classes over the C ABI.

Same class names, constructor arguments, getters and error behaviour as
``src/process/{ambiguity,clutter,detection}`` in the reference, so the parity tests read
like the reference's own unit tests (test/unit/process/ambiguity/TestAmbiguity.cpp).
Arrays replace the reference's containers: ``IqData`` -> 1-D complex arrays,
``Map<complex<double>>`` -> :class:`Map`, ``Detection`` -> :class:`Detection`.

Every ``process`` call runs CUDA kernels through libb200dd.so.  There is no CPU
fallback; missing library / device raises.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import capi


@dataclass
class Map:
    """Mirror of Map<std::complex<double>> (src/data/Map.h:30-42)."""
    data: np.ndarray  # [nRows = nDopplerBins][nCols = nDelayBins] complex128
    delay: np.ndarray  # int32 bins
    doppler: np.ndarray  # float64 Hz
    noisePower: float = 0.0
    maxPower: float = 0.0

    def get_nRows(self):
        return self.data.shape[0]

    def get_nCols(self):
        return self.data.shape[1]

    def to_json_km(self, timestamp, fs, device=-1) -> bytes:
        """delay_bin_to_km(to_json(timestamp), fs) (src/data/Map.cpp:116-185): the document blah2 sends on its map
        socket, rendered on the device from this map, its axes and its noisePower / maxPower."""
        mj = MapJson(self.delay, self.doppler, fs, device=device)
        try:
            return mj.render_host(self.data, self.noisePower, self.maxPower, timestamp)
        finally:
            mj.close()


@dataclass
class Detection:
    """Mirror of Detection (src/data/Detection.h:17-24)."""
    delay: np.ndarray
    doppler: np.ndarray
    snr: np.ndarray

    def get_nDetections(self):
        return int(self.delay.shape[0])


def _c128(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.complex128))


def _channel_count(name, x, y, dtypes, per_instant):
    """The instant count n of two contiguous channel buffers (numpy arrays or torch tensors) of a dtype in `dtypes`
    holding `per_instant` values per instant each; ValueError when they do not qualify or their counts differ."""
    counts = []
    for a in (x, y):
        torch_like = hasattr(a, "numel")
        dtype = str(a.dtype).replace("torch.", "")
        if dtype not in dtypes or not (a.is_contiguous() if torch_like else a.flags.c_contiguous):
            raise ValueError(f"{name}: channel buffers must be contiguous {' or '.join(dtypes)}, got {dtype}")
        size = a.numel() if torch_like else a.size
        if size % per_instant:
            raise ValueError(f"{name}: {size} values are not whole instants of {per_instant}")
        counts.append(size // per_instant)
    if counts[0] != counts[1]:
        raise ValueError(f"{name}: the channels hold {counts[0]} and {counts[1]} instants")
    return counts[0]


class _Handle:
    """Owner of one C-ABI handle: ``_lib`` and ``_h`` are set by the subclass's constructor, ``_destroy`` names the
    library function that frees ``_h``."""
    _destroy = None

    def close(self):
        if getattr(self, "_h", None):
            getattr(self._lib, self._destroy)(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _st(stream):
        """The stream argument of a call: the caller's stream, or NULL for the handle's own."""
        return capi.ptr(stream or None)


class Ambiguity(_Handle):
    """Ambiguity(delayMin, delayMax, dopplerMin, dopplerMax, fs, n, roundHamming=False)
    -- src/process/ambiguity/Ambiguity.h:34."""
    _destroy = "b200dd_caf_destroy"

    def __init__(self, delayMin, delayMax, dopplerMin, dopplerMax, fs, n, roundHamming=False, device=-1):
        lib = capi.load()
        p = capi.CafParams(int(delayMin), int(delayMax), int(dopplerMin), int(dopplerMax), int(fs), int(n),
                           int(bool(roundHamming)), int(device))
        h = C.c_void_p()
        capi.check(lib.b200dd_caf_create(C.byref(p), C.byref(h)))
        self._lib, self._h = lib, h
        g = capi.CafGeometry()
        capi.check(lib.b200dd_caf_get_geometry(h, C.byref(g)))
        self.geometry = g
        self.delay = np.empty(g.n_delay_bins, dtype=np.int32)
        self.doppler = np.empty(g.n_doppler_bins, dtype=np.float64)
        capi.check(lib.b200dd_caf_get_axes(h, capi.ptr(self.delay), capi.ptr(self.doppler)))
        self._n_samples = int(n)

    # getters, Ambiguity.h:46-58
    def get_doppler_middle(self):
        return self.geometry.doppler_middle

    def get_n_delay_bins(self):
        return self.geometry.n_delay_bins

    def get_n_doppler_bins(self):
        return self.geometry.n_doppler_bins

    def get_n_corr(self):
        return self.geometry.n_corr

    def get_cpi(self):
        return self.geometry.cpi

    def get_nfft(self):
        return self.geometry.nfft

    def get_n_samples(self):
        return self._n_samples

    @property
    def n_used(self):
        return self.geometry.n_used

    def process(self, x, y) -> Map:
        """Host path: x, y complex arrays (>= n_used samples).  Returns the Map; like the
        reference only the first nDopplerBins*nCorr samples are consumed and
        get_n_samples() afterwards reports that count (Ambiguity.cpp:105)."""
        x, y = _c128(x), _c128(y)
        if x.shape[0] != y.shape[0]:
            raise ValueError("x and y must have the same length")
        g = self.geometry
        out = np.empty((g.n_doppler_bins, g.n_delay_bins), dtype=np.complex128)
        capi.check(self._lib.b200dd_caf_process_host(self._h, capi.ptr(x), capi.ptr(y), x.shape[0], capi.ptr(out)))
        self._n_samples = g.n_used
        return Map(out, self.delay.copy(), self.doppler.copy())

    def process_device(self, d_x, d_y, d_map=None, stream=None):
        """Device path: torch complex64 CUDA tensors (or raw device pointers as ints).
        Asynchronous.  Returns None; result in d_map (or the handle's internal map)."""
        n = d_x.numel() if hasattr(d_x, "numel") else self.geometry.n_used
        capi.check(self._lib.b200dd_caf_process_device(self._h, capi.ptr(d_x), capi.ptr(d_y), int(n),
                                                       capi.ptr(d_map), self._st(stream)))

    def range_device(self, d_x, d_y, batch0, n_batches, d_R, stream=None):
        """Range stage on batches [batch0, batch0+n_batches): d_x, d_y hold exactly those batches."""
        capi.check(self._lib.b200dd_caf_range_device(self._h, capi.ptr(d_x), capi.ptr(d_y), int(batch0), int(n_batches),
                                                     capi.ptr(d_R), self._st(stream)))

    def doppler_device(self, d_R, col0, n_cols, d_map_tile, stream=None):
        """Doppler stage on delay columns [col0, col0+n_cols) of the complete range matrix d_R."""
        capi.check(self._lib.b200dd_caf_doppler_device(self._h, capi.ptr(d_R), int(col0), int(n_cols),
                                                       capi.ptr(d_map_tile), self._st(stream)))

    def place_tile(self, d_tile, col0, n_cols, d_map, stream=None):
        """Tile [nDop][n_cols] -> delay columns [col0, col0 + n_cols) of the row-major map d_map."""
        capi.check(self._lib.b200dd_caf_place_tile_device(self._h, capi.ptr(d_tile), int(col0), int(n_cols), capi.ptr(d_map),
                                                          self._st(stream)))

    def place_tiles(self, d_tiles, n_tiles, d_map, stream=None):
        """All gathered tiles of an equal column split (shard.block_range) -> the row-major map, one kernel."""
        capi.check(self._lib.b200dd_caf_place_tiles_device(self._h, capi.ptr(d_tiles), int(n_tiles), capi.ptr(d_map),
                                                           self._st(stream)))

    def profile_device(self, d_x, d_y, d_map=None, stream=None):
        """(ms_range, ms_doppler): CUDA-event durations of the two CAF kernels for one CPI."""
        a, b = C.c_float(), C.c_float()
        n = d_x.numel() if hasattr(d_x, "numel") else self.geometry.n_used
        capi.check(self._lib.b200dd_caf_profile_device(self._h, capi.ptr(d_x), capi.ptr(d_y), int(n), capi.ptr(d_map),
                                                       self._st(stream), C.byref(a), C.byref(b)))
        return a.value, b.value

    def debug_range_matrix(self):
        g = self.geometry
        out = np.empty((g.n_doppler_bins, g.n_delay_bins), dtype=np.complex64)
        capi.check(self._lib.b200dd_caf_debug_range_matrix(self._h, capi.ptr(out)))
        return out

    def device_map_ptr(self) -> int:
        return int(self._lib.b200dd_caf_device_map(self._h) or 0)

    def stream_ptr(self) -> int:
        return int(self._lib.b200dd_caf_stream(self._h) or 0)


class WienerHopf(_Handle):
    """WienerHopf(delayMin, delayMax, nSamples) -- src/process/clutter/WienerHopf.h:68."""
    _destroy = "b200dd_wh_destroy"

    def __init__(self, delayMin, delayMax, nSamples, device=-1):
        lib = capi.load()
        h = C.c_void_p()
        capi.check(lib.b200dd_wh_create(int(delayMin), int(delayMax), int(nSamples), int(device), C.byref(h)))
        self._lib, self._h = lib, h
        self.nSamples = int(nSamples)
        self.nBins = int(lib.b200dd_wh_n_bins(h))
        self.plan = capi.WhPlan()
        capi.check(lib.b200dd_wh_get_plan(h, C.byref(self.plan)))

    def process(self, x, y):
        """Host path.  Returns (ok, y_filtered): ok False <=> the reference returns false
        (Cholesky failure) and leaves y untouched (WienerHopf.cpp:111-122)."""
        x = _c128(x)
        y = _c128(y).copy()
        if x.shape[0] != self.nSamples or y.shape[0] != self.nSamples:
            raise ValueError("x and y must hold nSamples samples")
        rc = capi.check(self._lib.b200dd_wh_process_host(self._h, capi.ptr(x), capi.ptr(y)),
                        allow=(capi.FILTER_FAILED,))
        return rc == capi.OK, y

    def process_device(self, d_x, d_y, d_y_out=None, stream=None):
        out = d_y if d_y_out is None else d_y_out
        capi.check(self._lib.b200dd_wh_process_device(self._h, capi.ptr(d_x), capi.ptr(d_y), capi.ptr(out),
                                                      self._st(stream)))

    def profile_device(self, d_x, d_y, d_y_out, stream=None):
        """(ms_corr, ms_solve, ms_apply): CUDA-event durations of the filter's stages."""
        a, b, c = C.c_float(), C.c_float(), C.c_float()
        capi.check(self._lib.b200dd_wh_profile_device(self._h, capi.ptr(d_x), capi.ptr(d_y), capi.ptr(d_y_out),
                                                      self._st(stream), C.byref(a), C.byref(b),
                                                      C.byref(c)))
        return a.value, b.value, c.value

    def last_status(self) -> bool:
        rc = capi.check(self._lib.b200dd_wh_last_status(self._h), allow=(capi.FILTER_FAILED,))
        return rc == capi.OK

    def debug_weights(self):
        w = np.empty(self.nBins, dtype=np.complex128)
        a = np.empty(self.nBins, dtype=np.complex128)
        b = np.empty(self.nBins, dtype=np.complex128)
        capi.check(self._lib.b200dd_wh_debug_weights(self._h, capi.ptr(w), capi.ptr(a), capi.ptr(b)))
        return w, a, b


class WienerHopfChunk(_Handle):
    """The clutter filter on ONE CHUNK of a CPI that is split over several GPUs (SURVEY.md s8e row 3; C ABI
    b200dd_wh_create_chunk).  Device path only (complex64 CUDA tensors).  x_loc / y_loc are the chunk plus the
    halos `halos()` reports; blah2_b200.shard.wienerhopf_single_cpi_sharded drives it across ranks."""
    _destroy = "b200dd_wh_destroy"

    def __init__(self, delayMin, delayMax, nSamples, chunk_begin, chunk_len, device=-1):
        lib = capi.load()
        h = C.c_void_p()
        capi.check(lib.b200dd_wh_create_chunk(int(delayMin), int(delayMax), int(nSamples), int(chunk_begin), int(chunk_len),
                                              int(device), C.byref(h)))
        self._lib, self._h = lib, h
        self.nSamples, self.chunk_begin, self.chunk_len = int(nSamples), int(chunk_begin), int(chunk_len)
        self.nBins = int(lib.b200dd_wh_n_bins(h))
        a, b, c = C.c_uint32(), C.c_uint32(), C.c_uint32()
        capi.check(lib.b200dd_wh_chunk_halos(h, C.byref(a), C.byref(b), C.byref(c)))
        self.x_left, self.x_right, self.y_right = int(a.value), int(b.value), int(c.value)

    def halos(self):
        """(x_left, x_right, y_right) in samples."""
        return self.x_left, self.x_right, self.y_right

    def corr_device(self, d_x_loc, d_y_loc, d_ab, stream=None):
        """d_ab (complex128 CUDA tensor, 2 nBins) <- this chunk's share of (a, b)."""
        assert d_x_loc.numel() == self.x_left + self.chunk_len + self.x_right and d_y_loc.numel() == self.chunk_len + self.y_right
        capi.check(self._lib.b200dd_wh_chunk_corr_device(self._h, capi.ptr(d_x_loc), capi.ptr(d_y_loc), capi.ptr(d_ab),
                                                         self._st(stream)))

    def filter_device(self, d_ab, d_x_loc, d_y_loc, d_y_out, stream=None):
        """Replicated solve on the summed d_ab, then the chunk's chunk_len filtered samples into d_y_out."""
        assert d_y_out.numel() == self.chunk_len
        capi.check(self._lib.b200dd_wh_chunk_filter_device(self._h, capi.ptr(d_ab), capi.ptr(d_x_loc), capi.ptr(d_y_loc),
                                                           capi.ptr(d_y_out), self._st(stream)))

    def last_status(self) -> bool:
        rc = capi.check(self._lib.b200dd_wh_last_status(self._h), allow=(capi.FILTER_FAILED,))
        return rc == capi.OK

    def device_status(self) -> int:
        """Device pointer of the chunk's clutter-filter status word (0: the solve succeeded), written by filter_device.
        The solve is replicated, so every chunk's word holds the CPI's verdict (Pipeline.submit_map takes it)."""
        return int(self._lib.b200dd_wh_device_status(self._h))

    def debug_weights(self):
        """(w, a, b) of the last filter_device call (tests)."""
        w = np.empty(self.nBins, dtype=np.complex128)
        a = np.empty(self.nBins, dtype=np.complex128)
        b = np.empty(self.nBins, dtype=np.complex128)
        capi.check(self._lib.b200dd_wh_debug_weights(self._h, capi.ptr(w), capi.ptr(a), capi.ptr(b)))
        return w, a, b


class SpectrumAnalyser(_Handle):
    """SpectrumAnalyser(n, bandwidth) -- src/process/spectrum/SpectrumAnalyser.h:48.

    ``process(x)`` returns ``(spectrum, frequency)``: the two vectors the reference hands to
    ``IqData::update_spectrum`` / ``update_frequency`` (SpectrumAnalyser.cpp:55,68)."""
    _destroy = "b200dd_spectrum_destroy"

    def __init__(self, n, bandwidth, device=-1):
        lib = capi.load()
        h = C.c_void_p()
        capi.check(lib.b200dd_spectrum_create(int(n), float(bandwidth), int(device), C.byref(h)))
        self._lib, self._h = lib, h
        g = capi.SpectrumGeometry()
        capi.check(lib.b200dd_spectrum_get_geometry(h, C.byref(g)))
        self.geometry = g
        self.decimation, self.nSpectrum, self.nfft = int(g.decimation), int(g.n_spectrum), int(g.nfft)
        self.frequency = np.empty(int(g.n_frequency), dtype=np.float64)
        capi.check(lib.b200dd_spectrum_get_frequency(h, capi.ptr(self.frequency), int(g.n_frequency)))

    def process(self, x):
        """Host path: complex array with >= nfft samples (read, not consumed)."""
        x = _c128(x)
        out = np.empty(self.nSpectrum, dtype=np.complex128)
        capi.check(self._lib.b200dd_spectrum_process_host(self._h, capi.ptr(x), x.shape[0], capi.ptr(out)))
        return out, self.frequency.copy()

    def process_device(self, d_x, d_spectrum=None, stream=None):
        """Device path: torch complex64 (or complex128) CUDA tensor.  Asynchronous; pair with fetch()
        when d_spectrum is None."""
        n = d_x.numel()
        f64 = getattr(d_x, "element_size", lambda: 8)() == 16
        fn = self._lib.b200dd_spectrum_process_device_f64 if f64 else self._lib.b200dd_spectrum_process_device
        capi.check(fn(self._h, capi.ptr(d_x), int(n), capi.ptr(d_spectrum), self._st(stream)))

    def fold_slice_device(self, d_x, sample0, d_part, stream=None):
        """Folds the reference-channel samples [sample0, sample0 + len(d_x)) -- d_x a complex64 CUDA tensor whose first
        element is global sample sample0 -- into d_part (complex128 CUDA tensor of nSpectrum): their share of the
        CPI's spectrum before its last phase and transform.  Samples at or past nfft contribute nothing.
        Asynchronous; finish_device turns the parts of slices covering [0, nfft) into the spectrum."""
        n = int(d_x.numel())
        capi.check(self._lib.b200dd_spectrum_fold_slice_device(self._h, capi.ptr(d_x) if n else None, int(sample0), n,
                                                               capi.ptr(d_part), self._st(stream)))

    def finish_device(self, d_parts, d_spectrum=None, stream=None):
        """The spectrum from the parts of fold_slice_device (complex128 CUDA tensor [n_parts, nSpectrum]), summed in
        index order, into d_spectrum or, when None, the handle's buffer (read with fetch()).  Asynchronous."""
        n_parts = int(d_parts.numel()) // self.nSpectrum
        capi.check(self._lib.b200dd_spectrum_finish_device(self._h, capi.ptr(d_parts), n_parts, capi.ptr(d_spectrum),
                                                           self._st(stream)))

    def fetch(self, stream=None):
        out = np.empty(self.nSpectrum, dtype=np.complex128)
        capi.check(self._lib.b200dd_spectrum_fetch(self._h, capi.ptr(out), self._st(stream)))
        return out

    def profile_device(self, d_x, stream=None):
        """(ms_fold, ms_rest): CUDA-event durations of the folding pass and of reduction + DFT."""
        a, b = C.c_float(), C.c_float()
        capi.check(self._lib.b200dd_spectrum_profile_device(self._h, capi.ptr(d_x), int(d_x.numel()),
                                                            self._st(stream), C.byref(a),
                                                            C.byref(b)))
        return a.value, b.value


class _DetHandle(_Handle):
    """One b200dd_det handle shared by the three detection classes of a pipeline."""
    _destroy = "b200dd_det_destroy"

    def __init__(self, pfa=1e-5, nGuard=0, nTrain=0, minDelay=0, minDoppler=0.0, nCentroidDelay=0,
                 nCentroidDoppler=0, resolutionDoppler=1.0, doDelay=True, doDoppler=True, max_doppler_bins=8192,
                 max_delay_bins=2048, device=-1):
        lib = capi.load()
        p = capi.DetParams(float(pfa), int(nGuard), int(nTrain), int(minDelay), float(minDoppler),
                           int(nCentroidDelay), int(nCentroidDoppler), float(resolutionDoppler), int(bool(doDelay)),
                           int(bool(doDoppler)), int(device))
        h = C.c_void_p()
        capi.check(lib.b200dd_det_create(C.byref(p), int(max_doppler_bins), int(max_delay_bins), C.byref(h)))
        self._lib, self._h = lib, h
        self.cap = min(int(max_doppler_bins) * int(max_delay_bins), 1 << 18)

    def _bufs(self, cap):
        return [np.empty(max(1, cap), dtype=np.float64) for _ in range(3)]

    def process_map(self, m: Map, last_stage: int) -> Detection:
        data = _c128(m.data)
        delay = np.ascontiguousarray(m.delay, dtype=np.int32)
        doppler = np.ascontiguousarray(m.doppler, dtype=np.float64)
        od, of, os_ = self._bufs(self.cap)
        n = C.c_uint32()
        capi.check(self._lib.b200dd_det_process_host(self._h, last_stage, capi.ptr(data), data.shape[0],
                                                     data.shape[1], capi.ptr(delay), capi.ptr(doppler),
                                                     float(m.noisePower), capi.ptr(od), capi.ptr(of), capi.ptr(os_),
                                                     self.cap, C.byref(n)))
        k = n.value
        return Detection(od[:k].copy(), of[:k].copy(), os_[:k].copy())

    def process_device_map(self, d_map, nDop, nDel, delay, doppler, noisePower, last_stage, stream=None) -> Detection:
        delay = np.ascontiguousarray(delay, dtype=np.int32)
        doppler = np.ascontiguousarray(doppler, dtype=np.float64)
        od, of, os_ = self._bufs(self.cap)
        n = C.c_uint32()
        capi.check(self._lib.b200dd_det_process_device(self._h, last_stage, capi.ptr(d_map), int(nDop), int(nDel),
                                                       capi.ptr(delay), capi.ptr(doppler), float(noisePower),
                                                       capi.ptr(od), capi.ptr(of), capi.ptr(os_), self.cap,
                                                       C.byref(n), self._st(stream)))
        k = n.value
        return Detection(od[:k].copy(), of[:k].copy(), os_[:k].copy())

    def set_metrics_device(self, d_map, nDop, nDel, stream=None):
        out = np.empty(2, dtype=np.float64)
        capi.check(self._lib.b200dd_det_set_metrics_device(self._h, capi.ptr(d_map), int(nDop), int(nDel),
                                                           capi.ptr(out), self._st(stream)))
        return float(out[0]), float(out[1])

    def centroid(self, det: Detection) -> Detection:
        d = np.ascontiguousarray(det.delay, dtype=np.float64)
        f = np.ascontiguousarray(det.doppler, dtype=np.float64)
        s = np.ascontiguousarray(det.snr, dtype=np.float64)
        cap = max(1, d.shape[0])
        od, of, os_ = self._bufs(cap)
        n = C.c_uint32()
        capi.check(self._lib.b200dd_det_centroid_host(self._h, capi.ptr(d), capi.ptr(f), capi.ptr(s), d.shape[0],
                                                      capi.ptr(od), capi.ptr(of), capi.ptr(os_), cap, C.byref(n)))
        k = n.value
        return Detection(od[:k].copy(), of[:k].copy(), os_[:k].copy())

    def interpolate(self, det: Detection, m: Map) -> Detection:
        d = np.ascontiguousarray(det.delay, dtype=np.float64)
        f = np.ascontiguousarray(det.doppler, dtype=np.float64)
        s = np.ascontiguousarray(det.snr, dtype=np.float64)
        data = _c128(m.data)
        delay = np.ascontiguousarray(m.delay, dtype=np.int32)
        doppler = np.ascontiguousarray(m.doppler, dtype=np.float64)
        cap = max(1, d.shape[0])
        od, of, os_ = self._bufs(cap)
        n = C.c_uint32()
        capi.check(self._lib.b200dd_det_interpolate_host(self._h, capi.ptr(d), capi.ptr(f), capi.ptr(s), d.shape[0],
                                                         capi.ptr(data), data.shape[0], data.shape[1],
                                                         capi.ptr(delay), capi.ptr(doppler), float(m.noisePower),
                                                         capi.ptr(od), capi.ptr(of), capi.ptr(os_), cap, C.byref(n)))
        k = n.value
        return Detection(od[:k].copy(), of[:k].copy(), os_[:k].copy())


class CfarDetector1D:
    """CfarDetector1D(pfa, nGuard, nTrain, minDelay, minDoppler) -- CfarDetector1D.h:46."""

    def __init__(self, pfa, nGuard, nTrain, minDelay, minDoppler, max_doppler_bins=8192, max_delay_bins=2048,
                 device=-1):
        self._d = _DetHandle(pfa=pfa, nGuard=nGuard, nTrain=nTrain, minDelay=minDelay, minDoppler=minDoppler,
                             max_doppler_bins=max_doppler_bins, max_delay_bins=max_delay_bins, device=device)

    def process(self, m: Map) -> Detection:
        return self._d.process_map(m, capi.DET_CFAR)


class Centroid:
    """Centroid(nDelay, nDoppler, resolutionDoppler) -- Centroid.h:35."""

    def __init__(self, nDelay, nDoppler, resolutionDoppler, device=-1):
        self._d = _DetHandle(nCentroidDelay=nDelay, nCentroidDoppler=nDoppler, resolutionDoppler=resolutionDoppler,
                             max_doppler_bins=512, max_delay_bins=512, device=device)

    def process(self, det: Detection) -> Detection:
        return self._d.centroid(det)


class Interpolate:
    """Interpolate(doDelay, doDoppler) -- Interpolate.h:36."""

    def __init__(self, doDelay, doDoppler, max_doppler_bins=8192, max_delay_bins=2048, device=-1):
        self._d = _DetHandle(doDelay=doDelay, doDoppler=doDoppler, max_doppler_bins=max_doppler_bins,
                             max_delay_bins=max_delay_bins, device=device)

    def process(self, det: Detection, m: Map) -> Detection:
        return self._d.interpolate(det, m)


def set_metrics(m: Map) -> Map:
    """Map::set_metrics (Map.cpp:188-206) evaluated on the GPU for a host Map."""
    import torch  # device memory plumbing only

    d = _DetHandle(max_doppler_bins=m.data.shape[0], max_delay_bins=m.data.shape[1])
    t = torch.from_numpy(np.ascontiguousarray(m.data.astype(np.complex64))).cuda()
    m.noisePower, m.maxPower = d.set_metrics_device(t, m.data.shape[0], m.data.shape[1])
    torch.cuda.synchronize()
    d.close()
    return m


class MapJson(_Handle):
    """The map document of blah2.cpp:303-304 for maps of one shape: ``render_host`` for a complex128 host map,
    ``render_device`` + ``fetch`` for a device map (float2 / complex64, or complex128).  Raises B200ddError with
    code ERR_NONFINITE for a map cell with |z| = 0, inf or NaN, which has no JSON text."""
    _destroy = "b200dd_mapjson_destroy"

    def __init__(self, delay, doppler, fs, device=-1):
        lib = capi.load()
        self.delay = np.ascontiguousarray(np.asarray(delay, dtype=np.int32))
        self.doppler = np.ascontiguousarray(np.asarray(doppler, dtype=np.float64))
        h = C.c_void_p()
        capi.check(lib.b200dd_mapjson_create(self.doppler.size, self.delay.size, capi.ptr(self.delay),
                                             capi.ptr(self.doppler), int(fs), int(device), C.byref(h)))
        self._lib, self._h = lib, h
        self.max_bytes = int(lib.b200dd_mapjson_max_bytes(h))
        self._out = np.empty(self.max_bytes, dtype=np.uint8)

    def render_host(self, data, noisePower, maxPower, timestamp) -> bytes:
        data = _c128(data)
        if data.shape != (self.doppler.size, self.delay.size):
            raise ValueError(f"map shape {data.shape} != {(self.doppler.size, self.delay.size)}")
        n = C.c_size_t()
        capi.check(self._lib.b200dd_mapjson_render_host(self._h, capi.ptr(data), float(noisePower), float(maxPower),
                                                        int(timestamp), capi.ptr(self._out), self._out.size,
                                                        C.byref(n)))
        return self._out[:n.value].tobytes()

    def render_device(self, d_map, noisePower, maxPower, stream=None):
        """Asynchronous: d_map is a torch tensor [nDop, nDel] of complex64 / complex128 (or a float view of it)."""
        import torch
        f64 = d_map.dtype in (torch.complex128, torch.float64)
        capi.check(self._lib.b200dd_mapjson_render_device(self._h, capi.ptr(d_map), int(f64), float(noisePower),
                                                          float(maxPower), self._st(stream)))

    def fetch(self, timestamp, stream=None) -> bytes:
        n = C.c_size_t()
        capi.check(self._lib.b200dd_mapjson_fetch(self._h, int(timestamp), capi.ptr(self._out), self._out.size,
                                                  C.byref(n), self._st(stream)))
        return self._out[:n.value].tobytes()

    def cell_values(self, d_map, noisePower):
        """The double of every cell as the render computes it (10 log10|z| - noisePower), float64 [nDop, nDel]."""
        import torch
        f64 = d_map.dtype in (torch.complex128, torch.float64)
        out = torch.empty((self.doppler.size, self.delay.size), dtype=torch.float64, device=d_map.device)
        capi.check(self._lib.b200dd_mapjson_debug_cell_values(self._h, capi.ptr(d_map), int(f64), float(noisePower),
                                                              capi.ptr(out), None))
        torch.cuda.synchronize(d_map.device)
        return out.cpu().numpy()


class MaxHold(_Handle):
    """The max-hold map document blah2's API serves at /stash/map (api/stash/maxhold.js): per cell the maximum
    over the last 20 accepted CPIs, with the latest one's header.  ``push_device`` adds a CPI's device map
    (complex64 or complex128) with its set_metrics values; ``fetch`` renders the document.  ``fetch`` raises
    B200ddError with code ERR_NONFINITE when the last push was rejected (a cell or metric without JSON text) and
    ERR_ARG when nothing is held yet."""
    _destroy = "b200dd_maxhold_destroy"

    def __init__(self, delay, doppler, fs, device=-1):
        lib = capi.load()
        self.delay = np.ascontiguousarray(np.asarray(delay, dtype=np.int32))
        self.doppler = np.ascontiguousarray(np.asarray(doppler, dtype=np.float64))
        h = C.c_void_p()
        capi.check(lib.b200dd_maxhold_create(self.doppler.size, self.delay.size, capi.ptr(self.delay),
                                             capi.ptr(self.doppler), int(fs), int(device), C.byref(h)))
        self._lib, self._h = lib, h
        self.max_bytes = int(lib.b200dd_maxhold_max_bytes(h))
        self._out = np.empty(self.max_bytes, dtype=np.uint8)

    def push_device(self, d_map, noisePower, maxPower, stream=None):
        """Asynchronous: d_map is a torch tensor [nDop, nDel] of complex64 / complex128 (or a float view of it)."""
        import torch
        f64 = d_map.dtype in (torch.complex128, torch.float64)
        capi.check(self._lib.b200dd_maxhold_push_device(self._h, capi.ptr(d_map), int(f64), float(noisePower),
                                                        float(maxPower), self._st(stream)))

    def fetch(self, timestamp, stream=None) -> bytes:
        n = C.c_size_t()
        capi.check(self._lib.b200dd_maxhold_fetch(self._h, int(timestamp), capi.ptr(self._out), self._out.size,
                                                  C.byref(n), self._st(stream)))
        return self._out[:n.value].tobytes()


class DetectionJson(_Handle):
    """The detection document of blah2.cpp:312-317 and the API's /stash/detection history (api/stash/detection.js)
    of up to ``max_held`` detections.  ``render_device`` renders a device detection list (float64 tensors, the count
    in a uint32 / int32 device word); ``fetch`` writes its document and commits it to the history;
    ``fetch_stash`` writes the history.  ``render_host`` needs no handle and no device.  Raises B200ddError with code
    ERR_NONFINITE for a value without JSON text, ERR_CAPACITY for more than 2^18 detections or an overflowed history
    (see include/b200dd.h)."""
    _destroy = "b200dd_detjson_destroy"

    def __init__(self, fs, max_held=1 << 20, device=-1):
        lib = capi.load()
        h = C.c_void_p()
        capi.check(lib.b200dd_detjson_create(int(fs), int(max_held), int(device), C.byref(h)))
        self._lib, self._h = lib, h
        self.fs = int(fs)
        self.max_bytes = int(lib.b200dd_detjson_max_bytes(h))
        self.stash_max_bytes = int(lib.b200dd_detjson_stash_max_bytes(h))
        self._out = np.empty(self.max_bytes, dtype=np.uint8)
        self._stash = np.empty(self.stash_max_bytes, dtype=np.uint8)

    def render_device(self, d_delay, d_doppler, d_snr, d_count, stream=None):
        """Asynchronous: the three lists are float64 device tensors, d_count a one-word device tensor."""
        capi.check(self._lib.b200dd_detjson_render_device(self._h, capi.ptr(d_delay), capi.ptr(d_doppler),
                                                          capi.ptr(d_snr), capi.ptr(d_count),
                                                          self._st(stream)))

    def fetch(self, timestamp, stream=None) -> bytes:
        n = C.c_size_t()
        capi.check(self._lib.b200dd_detjson_fetch(self._h, int(timestamp), capi.ptr(self._out), self._out.size,
                                                  C.byref(n), self._st(stream)))
        return self._out[:n.value].tobytes()

    def fetch_stash(self, stream=None) -> bytes:
        n = C.c_size_t()
        capi.check(self._lib.b200dd_detjson_fetch_stash(self._h, capi.ptr(self._stash), self._stash.size, C.byref(n),
                                                        self._st(stream)))
        return self._stash[:n.value].tobytes()

    @staticmethod
    def render_host(delay, doppler, snr, timestamp, fs) -> bytes:
        """Detection::delay_bin_to_km(Detection::to_json(timestamp), fs) of host lists, on the CPU."""
        lib = capi.load()
        v = [np.ascontiguousarray(np.asarray(a, dtype=np.float64).ravel()) for a in (delay, doppler, snr)]
        if not v[0].size == v[1].size == v[2].size:
            raise ValueError("delay, doppler and snr differ in length")
        out = np.empty(80 + 75 * v[0].size, dtype=np.uint8)
        n = C.c_size_t()
        capi.check(lib.b200dd_detjson_render_host(capi.ptr(v[0]), capi.ptr(v[1]), capi.ptr(v[2]), v[0].size,
                                                  int(timestamp), int(fs), capi.ptr(out), out.size, C.byref(n)))
        return out[:n.value].tobytes()


class IqDataJson(_Handle):
    """The IQ-data document of blah2.cpp:299-300 (IqData::to_json of the spectrum) and the API's /stash/iqdata history
    of the last 20 documents (api/stash/iqdata.js).  ``min``, ``max`` and ``mean`` are the IqData members the document
    carries (blah2 never assigns them); they must be finite.  ``render_device`` renders a device spectrum (a complex128
    tensor of ``n_spectrum`` bins); ``fetch`` writes its document and commits it to the history; ``fetch_stash`` writes
    the history.  ``render_host`` needs no handle and no device.  Raises B200ddError with code ERR_NONFINITE for a
    bin that is zero, infinite or NaN (see include/b200dd.h)."""
    _destroy = "b200dd_iqjson_destroy"

    def __init__(self, n_spectrum, min, max, mean, device=-1):
        lib = capi.load()
        h = C.c_void_p()
        capi.check(lib.b200dd_iqjson_create(int(n_spectrum), float(min), float(max), float(mean), int(device),
                                            C.byref(h)))
        self._lib, self._h = lib, h
        self.n_spectrum = int(n_spectrum)
        self.metrics = (float(min), float(max), float(mean))
        self.max_bytes = int(lib.b200dd_iqjson_max_bytes(h))
        self.stash_max_bytes = int(lib.b200dd_iqjson_stash_max_bytes(h))
        self._out = np.empty(self.max_bytes, dtype=np.uint8)
        self._stash = np.empty(self.stash_max_bytes, dtype=np.uint8)

    def render_device(self, d_spectrum, stream=None):
        """Asynchronous: d_spectrum is a complex128 device tensor of n_spectrum bins."""
        capi.check(self._lib.b200dd_iqjson_render_device(self._h, capi.ptr(d_spectrum),
                                                         self._st(stream)))

    def fetch(self, timestamp, stream=None) -> bytes:
        n = C.c_size_t()
        capi.check(self._lib.b200dd_iqjson_fetch(self._h, int(timestamp), capi.ptr(self._out), self._out.size,
                                                 C.byref(n), self._st(stream)))
        return self._out[:n.value].tobytes()

    def fetch_stash(self, stream=None) -> bytes:
        n = C.c_size_t()
        capi.check(self._lib.b200dd_iqjson_fetch_stash(self._h, capi.ptr(self._stash), self._stash.size, C.byref(n),
                                                       self._st(stream)))
        return self._stash[:n.value].tobytes()

    def bin_values(self, d_spectrum):
        """The double of every bin, 10 log10|s| as the device render computes it (a test aid)."""
        import torch
        out = torch.empty(self.n_spectrum, dtype=torch.float64, device=d_spectrum.device)
        capi.check(self._lib.b200dd_iqjson_debug_bin_values(self._h, capi.ptr(d_spectrum), capi.ptr(out), None))
        torch.cuda.synchronize(d_spectrum.device)
        return out.cpu().numpy()

    @staticmethod
    def render_host(spectrum, min, max, mean, timestamp) -> bytes:
        """IqData::to_json(timestamp) of host complex bins, on the CPU."""
        lib = capi.load()
        s = np.ascontiguousarray(np.asarray(spectrum, dtype=np.complex128).ravel())
        out = np.empty(160 + 25 * s.size, dtype=np.uint8)
        n = C.c_size_t()
        capi.check(lib.b200dd_iqjson_render_host(capi.ptr(s), s.size, float(min), float(max), float(mean),
                                                 int(timestamp), capi.ptr(out), out.size, C.byref(n)))
        return out[:n.value].tobytes()


def timing_render_host(t_start, t_now, n, names, values) -> bytes:
    """blah2's Timing(t_start), update(t_now, values, names) after n - 1 earlier updates, then to_json(), on the CPU
    (b200dd_timing_render_host).  Raises B200ddError (ERR_ARG) for a name written unescaped or a non-finite value."""
    lib = capi.load()
    v = np.ascontiguousarray(np.asarray(values, dtype=np.float64).ravel())
    if len(names) != v.size:
        raise ValueError("names and values differ in length")
    arr = (C.c_char_p * max(v.size, 1))(*[s.encode() if isinstance(s, str) else s for s in names])
    out = np.empty(int(lib.b200dd_timing_max_bytes()), dtype=np.uint8)
    nb = C.c_size_t()
    capi.check(lib.b200dd_timing_render_host(int(t_start), int(t_now), int(n), arr, capi.ptr(v), v.size,
                                             capi.ptr(out), out.size, C.byref(nb)))
    return out[:nb.value].tobytes()


def _fetch_growing(buf, call):
    """call(buf) -> (rc, n_bytes); a too-small buffer is grown to the reported size and the call repeated."""
    rc, n = call(buf)
    if rc == capi.ERR_CAPACITY and n > buf.size:
        buf = np.empty(n, dtype=np.uint8)
        rc, n = call(buf)
    capi.check(rc)
    return buf, buf[:n].tobytes()


class Tracker(_Handle):
    """blah2's Tracker (src/process/tracker/Tracker.cpp) with its tracks on the device, named like the reference's
    constructor Tracker(m, n, nDelete, cpi, maxAccInit, rangeRes, lambda) with rangeRes = c / fs and lambda = c / fc
    given as fs and fc (blah2.cpp:193-195).  ``process_device`` / ``process_host`` run Tracker::process on one CPI's
    detections; ``fetch`` returns Track::to_json(timestamp).  ``max_tracks`` and ``max_history`` bound the state: past
    them fetch raises ERR_CAPACITY until ``reset``.  A non-finite track value raises ERR_NONFINITE at fetch."""
    _destroy = "b200dd_tracker_destroy"

    def __init__(self, m, n, nDelete, cpi, maxAcc, fs, fc, max_tracks=1 << 16, max_history=64, device=-1):
        lib = capi.load()
        self.params = capi.TrackerParams(int(m), int(n), int(nDelete), float(cpi), float(maxAcc), int(fs), int(fc))
        h = C.c_void_p()
        capi.check(lib.b200dd_tracker_create(C.byref(self.params), int(max_tracks), int(max_history), int(device),
                                             C.byref(h)))
        self._lib, self._h = lib, h
        self.max_bytes = int(lib.b200dd_tracker_max_bytes(h))
        self._out = np.empty(1 << 16, dtype=np.uint8)

    def process_device(self, d_delay, d_doppler, d_snr, d_count, timestamp, stream=None):
        """Asynchronous: the lists are float64 device tensors, d_count a one-word device tensor."""
        capi.check(self._lib.b200dd_tracker_process_device(self._h, capi.ptr(d_delay), capi.ptr(d_doppler),
                                                           capi.ptr(d_snr), capi.ptr(d_count), int(timestamp),
                                                           self._st(stream)))

    def process_host(self, delay, doppler, snr, timestamp, stream=None):
        v = [np.ascontiguousarray(np.asarray(a, dtype=np.float64).ravel()) for a in (delay, doppler, snr)]
        if not v[0].size == v[1].size == v[2].size:
            raise ValueError("delay, doppler and snr differ in length")
        capi.check(self._lib.b200dd_tracker_process_host(self._h, capi.ptr(v[0]), capi.ptr(v[1]), capi.ptr(v[2]),
                                                         v[0].size, int(timestamp),
                                                         self._st(stream)))

    def fetch(self, timestamp, stream=None) -> bytes:
        def call(buf):
            n = C.c_size_t()
            rc = self._lib.b200dd_tracker_fetch(self._h, int(timestamp), capi.ptr(buf), buf.size, C.byref(n),
                                                self._st(stream))
            return rc, n.value
        self._out, doc = _fetch_growing(self._out, call)
        return doc

    def reset(self):
        capi.check(self._lib.b200dd_tracker_reset(self._h))

    def reserve(self, max_tracks, max_history, stream=None):
        """Raise the limits to at least max_tracks x max_history, keeping every track (b200dd_tracker_reserve)."""
        capi.check(self._lib.b200dd_tracker_reserve(self._h, int(max_tracks), int(max_history), self._st(stream)))
        self.max_bytes = int(self._lib.b200dd_tracker_max_bytes(self._h))

    def usage(self, stream=None):
        """(live tracks, longest history among them) after the work enqueued so far (synchronous)."""
        live, longest = C.c_uint32(), C.c_uint32()
        capi.check(self._lib.b200dd_tracker_usage(self._h, C.byref(live), C.byref(longest), self._st(stream)))
        return live.value, longest.value


def record_bytes(max_detections, n_spectrum=0, timing=False, detection=True) -> int:
    """The size of a pipeline's CPI record (b200dd_pipeline_enable_export): a 64-byte header, 80 bytes of stage stamps
    with the timing stage, 16 bytes per spectrum bin with the spectrum stage and 24 bytes per detection slot with
    detection, rounded up to 16 bytes."""
    n = 64 + (80 if timing else 0) + 16 * int(n_spectrum) + (24 * int(max_detections) if detection else 0)
    return (n + 15) // 16 * 16


class _DeviceBytes:
    """A device byte range as torch.as_tensor takes it (__cuda_array_interface__), without a copy."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False),
                                         "version": 3}


class Pipeline(_Handle):
    """One CPI through the body of the reference's process thread (src/blah2.cpp:268-287):
    [WienerHopf] -> Ambiguity -> Map::set_metrics -> [CfarDetector1D -> Centroid -> Interpolate],
    intermediates resident on the device.  Parameters are named like config/config.yml."""
    _destroy = "b200dd_pipeline_destroy"

    def __init__(self, delayMin, delayMax, dopplerMin, dopplerMax, fs, nSamples, roundHamming=True, clutter=None,
                 detection=None, device=-1, max_detections=4096, spectrum_bandwidth=None, map_json=False,
                 maxhold=False, detection_json=False, max_held_detections=1 << 20, tracker=None, max_tracks=1 << 16,
                 max_track_history=64):
        lib = capi.load()
        p = capi.PipelineParams()
        p.caf = capi.CafParams(int(delayMin), int(delayMax), int(dopplerMin), int(dopplerMax), int(fs),
                               int(nSamples), int(bool(roundHamming)), int(device))
        p.clutter_enable = int(clutter is not None)
        if clutter is not None:
            p.clutter_delay_min, p.clutter_delay_max = int(clutter[0]), int(clutter[1])
        p.detection_enable = int(detection is not None)
        d = detection or {}
        tcpi = float(nSamples) / float(fs)
        p.det = capi.DetParams(float(d.get("pfa", 1e-5)), int(d.get("nGuard", 2)), int(d.get("nTrain", 6)),
                               int(d.get("minDelay", 5)), float(d.get("minDoppler", 15.0)),
                               int(d.get("nCentroid", 6)), int(d.get("nCentroid", 6)), 1.0 / tcpi, 1, 1, int(device))
        h = C.c_void_p()
        capi.check(lib.b200dd_pipeline_create(C.byref(p), C.byref(h)))
        self._lib, self._h = lib, h
        g = capi.CafGeometry()
        capi.check(lib.b200dd_pipeline_get_geometry(h, C.byref(g)))
        self.geometry = g
        self.delay = np.empty(g.n_delay_bins, dtype=np.int32)
        self.doppler = np.empty(g.n_doppler_bins, dtype=np.float64)
        capi.check(lib.b200dd_pipeline_get_axes(h, capi.ptr(self.delay), capi.ptr(self.doppler)))
        self.cap = int(max_detections)
        self._od, self._of, self._os = (np.empty(self.cap, dtype=np.float64) for _ in range(3))
        self.n_samples = int(nSamples)
        self.n_spectrum = 0
        if spectrum_bandwidth is not None:  # spectrumAnalyser->process(x), blah2.cpp:263-265
            ns = C.c_uint32()
            capi.check(lib.b200dd_pipeline_enable_spectrum(h, float(spectrum_bandwidth), C.byref(ns)))
            self.n_spectrum = int(ns.value)
        self.map_json_max_bytes = 0
        if map_json:  # map->to_json + delay_bin_to_km for every CPI, blah2.cpp:303-304
            mb = C.c_size_t()
            capi.check(lib.b200dd_pipeline_enable_map_json(h, C.byref(mb)))
            self.map_json_max_bytes = int(mb.value)
        self._json = np.empty(max(self.map_json_max_bytes, 1), dtype=np.uint8)
        self.maxhold_max_bytes = 0
        if maxhold:  # the API's /stash/map window over the last 20 CPIs, api/stash/maxhold.js
            mb = C.c_size_t()
            capi.check(lib.b200dd_pipeline_enable_maxhold(h, C.byref(mb)))
            self.maxhold_max_bytes = int(mb.value)
        self._maxhold = np.empty(max(self.maxhold_max_bytes, 1), dtype=np.uint8)
        self.detection_json_max_bytes = self.detection_stash_max_bytes = 0
        if detection_json:  # detection->to_json + delay_bin_to_km, blah2.cpp:312-317, and /stash/detection
            db, sb = C.c_size_t(), C.c_size_t()
            capi.check(lib.b200dd_pipeline_enable_detection_json(h, int(max_held_detections), C.byref(db),
                                                                 C.byref(sb)))
            self.detection_json_max_bytes, self.detection_stash_max_bytes = int(db.value), int(sb.value)
        self._detjson = np.empty(max(self.detection_json_max_bytes, 1), dtype=np.uint8)
        self._detstash = np.empty(max(self.detection_stash_max_bytes, 1), dtype=np.uint8)
        self.track_max_bytes = 0
        if tracker is not None:  # tracker->process + track->to_json, blah2.cpp:291-296 and :324-328
            t = tracker
            tp = capi.TrackerParams(int(t.get("M", 3)), int(t.get("N", 5)), int(t.get("delete", 10)), 0.0,
                                    float(t.get("maxAcc", 10)), 0, int(t["fc"]))  # cpi, fs: the pipeline's
            mb = C.c_size_t()
            capi.check(lib.b200dd_pipeline_enable_tracker(h, C.byref(tp), int(max_tracks), int(max_track_history),
                                                          C.byref(mb)))
            self.track_max_bytes = int(mb.value)
        self._track = np.empty(1 << 16, dtype=np.uint8)
        self.iqdata_json_max_bytes = self.iqdata_stash_max_bytes = 0  # see enable_iqdata_json
        self._iqjson = self._iqstash = np.empty(1, dtype=np.uint8)

    def _fetch_into(self, fn, buf, *args):
        """fn(handle, *args, buf, its size, &n), then the n bytes it wrote into buf."""
        n = C.c_size_t()
        capi.check(fn(self._h, *args, capi.ptr(buf), buf.size, C.byref(n)))
        return buf[:n.value].tobytes()

    def fetch_track_json(self, timestamp) -> bytes:
        """The track document after the last fetched CPI (call after fetch()): the first call per CPI runs the tracker
        on that CPI's detections with `timestamp`.  Raises B200ddError with code FILTER_FAILED when that CPI's
        clutter-filter solve failed and ERR_CAPACITY when CFAR overflowed the list (the tracker is unchanged), and
        ERR_CAPACITY / ERR_NONFINITE as Tracker.fetch."""
        def call(buf):
            n = C.c_size_t()
            rc = self._lib.b200dd_pipeline_fetch_track_json(self._h, int(timestamp), capi.ptr(buf), buf.size,
                                                            C.byref(n))
            return rc, n.value
        self._track, doc = _fetch_growing(self._track, call)
        return doc

    def fetch_detection_json(self, timestamp) -> bytes:
        """The detection document of the last fetched CPI (call after fetch()), committed to the /stash/detection
        history.  Raises B200ddError with code FILTER_FAILED when that CPI's clutter-filter solve failed (nothing is
        sent, the history is unchanged), ERR_CAPACITY when CFAR overflowed the list."""
        return self._fetch_into(self._lib.b200dd_pipeline_fetch_detection_json, self._detjson, int(timestamp))

    def fetch_detection_stash(self) -> bytes:
        """The /stash/detection document of the documents fetched so far."""
        return self._fetch_into(self._lib.b200dd_pipeline_fetch_detection_stash, self._detstash)

    def fetch_maxhold(self, timestamp) -> bytes:
        """The /stash/map document after the last fetched CPI (call after fetch()).  Raises B200ddError with code
        FILTER_FAILED when that CPI's clutter-filter solve failed (the window is unchanged), ERR_ARG when the stage
        is not enabled or nothing has been submitted."""
        return self._fetch_into(self._lib.b200dd_pipeline_fetch_maxhold, self._maxhold, int(timestamp))

    def fetch_map_json(self, timestamp) -> bytes:
        """The map document of the last fetched CPI (call after fetch()).  Raises B200ddError with code
        FILTER_FAILED when that CPI's clutter-filter solve failed: the reference sends no map then."""
        return self._fetch_into(self._lib.b200dd_pipeline_fetch_map_json, self._json, int(timestamp))

    def enable_iqdata_json(self, min, max, mean):
        """Renders the IQ-data document of every CPI submitted from now on (blah2.cpp:299-300), right after the spectrum
        stage, and keeps the /stash/iqdata history of the last 20 fetched documents, starting empty.  min, max and mean
        are the IqData members the document carries.  Needs ``spectrum_bandwidth``; enabling the spectrum stage again
        disables this stage."""
        db, sb = C.c_size_t(), C.c_size_t()
        capi.check(self._lib.b200dd_pipeline_enable_iqdata_json(self._h, float(min), float(max), float(mean),
                                                                C.byref(db), C.byref(sb)))
        self.iqdata_json_max_bytes, self.iqdata_stash_max_bytes = int(db.value), int(sb.value)
        self._iqjson = np.empty(self.iqdata_json_max_bytes, dtype=np.uint8)
        self._iqstash = np.empty(self.iqdata_stash_max_bytes, dtype=np.uint8)

    def fetch_iqdata_json(self, timestamp) -> bytes:
        """The IQ-data document of the last fetched CPI (call after fetch()), committed to the /stash/iqdata history.
        Raises B200ddError with code FILTER_FAILED when that CPI's clutter-filter solve failed (nothing is sent, the
        history is unchanged), ERR_NONFINITE when a spectrum bin has no text."""
        return self._fetch_into(self._lib.b200dd_pipeline_fetch_iqdata_json, self._iqjson, int(timestamp))

    def fetch_iqdata_stash(self) -> bytes:
        """The /stash/iqdata document of the documents fetched so far."""
        return self._fetch_into(self._lib.b200dd_pipeline_fetch_iqdata_stash, self._iqstash)

    def enable_timing_json(self, t_start):
        """Stamps every CPI submitted from now on at its stage boundaries on the device and builds blah2's timing
        document (blah2.cpp:331-345) from those stamps; keeps the /stash/timing history of the last 20 committed
        documents.  ``t_start`` is Timing's tStart (POSIX ms); nCpi and the history start at 0 and empty."""
        db, sb = C.c_size_t(), C.c_size_t()
        capi.check(self._lib.b200dd_pipeline_enable_timing_json(self._h, int(t_start), C.byref(db), C.byref(sb)))
        self.timing_json_max_bytes, self.timing_stash_max_bytes = int(db.value), int(sb.value)
        self._tmjson = np.empty(self.timing_json_max_bytes, dtype=np.uint8)
        self._tmstash = np.empty(self.timing_stash_max_bytes, dtype=np.uint8)
        if getattr(self, "export_max_detections", 0):  # the record now carries the stamps
            self.enable_export(self.export_max_detections)

    def fetch_timing_json(self, timestamp) -> bytes:
        """The timing document of the last fetched CPI with tNow = ``timestamp`` (call after fetch() and, with the
        tracker, after fetch_track_json()), committed to the /stash/timing history.  Raises B200ddError with code
        FILTER_FAILED when that CPI's clutter-filter solve failed (nothing is sent, nCpi and the history are
        unchanged), ERR_ARG when called too early or twice, or when a value has more than 15 significant digits (the
        document is then written but not committed; ``last_timing_doc`` holds it)."""
        n = C.c_size_t()
        rc = self._lib.b200dd_pipeline_fetch_timing_json(self._h, int(timestamp), capi.ptr(self._tmjson),
                                                         self._tmjson.size, C.byref(n))
        self.last_timing_doc = self._tmjson[:n.value].tobytes()
        capi.check(rc)
        return self.last_timing_doc

    def fetch_timing_stash(self) -> bytes:
        """The /stash/timing document of the documents committed so far."""
        return self._fetch_into(self._lib.b200dd_pipeline_fetch_timing_stash, self._tmstash)

    def timing_values(self):
        """The stage names and times (ms) behind the last timing document written (a test aid)."""
        names, values, count = (C.c_char_p * 16)(), np.empty(16, dtype=np.float64), C.c_uint32()
        capi.check(self._lib.b200dd_pipeline_debug_timing_values(self._h, names, capi.ptr(values), 16, C.byref(count)))
        return [names[i].decode() for i in range(count.value)], values[:count.value].copy()

    @staticmethod
    def share_history(pipes):
        """Makes the max-hold window, the detection and IQ-data histories and the tracker of ``pipes`` one object
        (b200dd_pipeline_share_history), for pipelines used alternately: after every fetch their stash and track
        documents are those of one pipeline given the same CPIs in submit order.  Each member then holds one unfetched
        CPI at a time, fetch() follows submit order across the set, and a member's CPI enters the max-hold window at
        its fetch().  The pipelines must have equal parameters and stages; the histories start empty.  Raises
        B200ddError (ERR_ARG) otherwise."""
        pipes = list(pipes)
        arr = (C.c_void_p * max(len(pipes), 1))(*[p._h for p in pipes])
        capi.check(capi.load().b200dd_pipeline_share_history(arr, len(pipes)))

    def enable_export(self, max_detections=4096) -> int:
        """Every CPI submitted from now on also packs its record: everything the fetches read besides the map, in
        one fixed-size device buffer (b200dd_pipeline_enable_export).  Detections past ``max_detections`` (1 .. 2^18)
        do not travel: such a CPI imports as a CFAR overflow.  Returns the record's size in bytes, kept as
        ``record_bytes`` (enable_timing_json afterwards packs the stamps too and updates it)."""
        nb = C.c_size_t()
        capi.check(self._lib.b200dd_pipeline_enable_export(self._h, int(max_detections), C.byref(nb)))
        self.export_max_detections, self.record_bytes = int(max_detections), int(nb.value)
        return self.record_bytes

    def export_record(self):
        """The last submit's record as a uint8 CUDA tensor of ``record_bytes`` that views the pipeline's buffer: valid
        until the next submit, written on that submit's stream."""
        import torch
        p = C.c_void_p()
        capi.check(self._lib.b200dd_pipeline_export_record(self._h, C.byref(p)))
        return torch.as_tensor(_DeviceBytes(int(p.value), self.record_bytes))

    def submit_record(self, d_record, d_map):
        """Takes the CPI another pipeline of the same parameters and spectrum / timing stages exported: its record
        and its complex64 map (device buffers, complete when this is called).  Then fetch() and every fetch_* behave
        as after a submit; d_map must stay untouched until fetch().  Raises B200ddError (ERR_ARG) for a record of
        other parameters or stages."""
        capi.check(self._lib.b200dd_pipeline_submit_record(self._h, capi.ptr(d_record), capi.ptr(d_map)))

    def submit_map(self, d_map, d_status=None, d_parts=None, stream=None):
        """Takes a CPI whose complex64 map d_map (nDoppler x nDelay CUDA tensor) was computed elsewhere -- e.g. placed
        from the tiles of shard.SingleCpiPlan -- and runs set_metrics, detection and every product after them on it
        (b200dd_pipeline_submit_map).  d_status: device pointer (int) of the clutter-filter verdict, required iff the
        clutter filter is enabled (WienerHopfChunk.device_status()); d_parts: the spectrum parts of
        SpectrumAnalyser.fold_slice_device as a complex128 CUDA tensor [n_parts, nSpectrum], required iff the spectrum
        stage is enabled.  Asynchronous on `stream`; then fetch() and every fetch_* behave as after a submit.  d_map
        must stay untouched until fetch().  Raises B200ddError (ERR_ARG) for a missing or unexpected argument."""
        n_parts = int(d_parts.numel()) // max(self.n_spectrum, 1) if d_parts is not None else 0
        capi.check(self._lib.b200dd_pipeline_submit_map(self._h, capi.ptr(d_map), capi.ptr(d_status), capi.ptr(d_parts),
                                                        n_parts, self._st(stream)))

    def stamp(self, slot, stream=None):
        """Timing stage: stamps the boundary ``slot`` (capi.STAMP_CHAIN, _SPECTRUM, _CLUTTER) of the CPI about to be
        given to submit_map, on ``stream``; boundaries not stamped are stamped at submit_map's start.  Does nothing
        when the timing stage is off."""
        capi.check(self._lib.b200dd_pipeline_stamp(self._h, int(slot), self._st(stream)))

    def fetch_spectrum(self):
        """Spectrum of the reference channel of the last submitted CPI (complex128, nSpectrum bins)."""
        out = np.empty(self.n_spectrum, dtype=np.complex128)
        capi.check(self._lib.b200dd_pipeline_fetch_spectrum(self._h, capi.ptr(out), self.n_spectrum))
        return out

    def _result(self, res, want_map_arr=None):
        skipped = res.filter_status != capi.OK
        # a failed clutter-filter solve skips the CPI (blah2.cpp:270-273): no detections, no metrics, no map product
        k = 0 if skipped else min(res.n_detections, self.cap)
        det = Detection(self._od[:k].copy(), self._of[:k].copy(), self._os[:k].copy())
        return dict(skipped=skipped, noisePower=res.noise_power, maxPower=res.max_power,
                    detections=det, map=None if skipped else want_map_arr)

    def process(self, x, y, want_map=True, map_out=None):
        """Host path: complex128 arrays (pinned torch tensors / numpy).  Synchronous."""
        g = self.geometry
        if map_out is None and want_map:
            map_out = np.empty((g.n_doppler_bins, g.n_delay_bins), dtype=np.complex128)
        n = x.numel() if hasattr(x, "numel") else x.shape[0]
        res = capi.CpiResult()
        capi.check(self._lib.b200dd_pipeline_process_host(self._h, capi.ptr(x), capi.ptr(y), int(n),
                                                          capi.ptr(map_out) if map_out is not None else None,
                                                          C.byref(res), capi.ptr(self._od), capi.ptr(self._of),
                                                          capi.ptr(self._os), self.cap), allow=(capi.ERR_CAPACITY,))
        return self._result(res, map_out)

    def submit_host(self, x, y, map_out=None):
        """Asynchronous host path: enqueue H2D + kernels + D2H(map) and return; pair with fetch().
        x, y, map_out must stay alive (pinned for real overlap) until fetch() returns."""
        n = x.numel() if hasattr(x, "numel") else x.shape[0]
        self._pending_map = map_out
        capi.check(self._lib.b200dd_pipeline_submit_host(self._h, capi.ptr(x), capi.ptr(y), int(n),
                                                         capi.ptr(map_out) if map_out is not None else None))

    def submit_host_rspduo(self, iq, map_out=None):
        """Asynchronous host path fed with the reference's replay layout: int16 [n, 4] = I1 Q1 I2 Q2
        (blah2_b200/scene.py write_rspduo).  Pair with fetch()."""
        n = (iq.numel() if hasattr(iq, "numel") else iq.size) // 4
        self._pending_map = map_out
        capi.check(self._lib.b200dd_pipeline_submit_host_rspduo(self._h, capi.ptr(iq), int(n),
                                                                capi.ptr(map_out) if map_out is not None else None))

    def submit_host_ci8(self, x_iq, y_iq, map_out=None):
        """Asynchronous host path fed with HackRF's / Kraken's format: reference and surveillance channel as two int8
        arrays or tensors of 2n values (or shape (n, 2)), interleaved I, Q.  A uint8 buffer (rtl-sdr's bytes) is read
        as int8, as blah2's Kraken source does: no offset is removed.  Pair with fetch(); the buffers must stay alive
        (pinned for real overlap) until fetch() returns."""
        n = _channel_count("submit_host_ci8", x_iq, y_iq, ("int8", "uint8"), 2)
        self._pending_map = map_out
        capi.check(self._lib.b200dd_pipeline_submit_host_ci8(self._h, capi.ptr(x_iq), capi.ptr(y_iq), int(n),
                                                             capi.ptr(map_out) if map_out is not None else None))

    def submit_host_cf32(self, x, y, map_out=None):
        """Asynchronous host path fed with USRP's format: reference and surveillance channel as two complex64 arrays
        or tensors of n samples.  Pair with fetch(), lifetimes as submit_host_ci8."""
        n = _channel_count("submit_host_cf32", x, y, ("complex64",), 1)
        self._pending_map = map_out
        capi.check(self._lib.b200dd_pipeline_submit_host_cf32(self._h, capi.ptr(x), capi.ptr(y), int(n),
                                                              capi.ptr(map_out) if map_out is not None else None))

    def submit_device(self, d_x, d_y, d_map=None, stream=None):
        n = d_x.numel() if hasattr(d_x, "numel") else self.n_samples
        capi.check(self._lib.b200dd_pipeline_submit_device(self._h, capi.ptr(d_x), capi.ptr(d_y), int(n),
                                                           capi.ptr(d_map), self._st(stream)))

    def prepare_device(self, d_x, d_y, d_map=None, stream=None):
        """Plan creation for submit_device on this buffer triple (records the CUDA graph of the chain now)."""
        n = d_x.numel() if hasattr(d_x, "numel") else self.n_samples
        capi.check(self._lib.b200dd_pipeline_prepare_device(self._h, capi.ptr(d_x), capi.ptr(d_y), int(n),
                                                            capi.ptr(d_map), self._st(stream)))

    def fetch(self, stream=None):
        res = capi.CpiResult()
        capi.check(self._lib.b200dd_pipeline_fetch(self._h, C.byref(res), capi.ptr(self._od), capi.ptr(self._of),
                                                   capi.ptr(self._os), self.cap,
                                                   self._st(stream)), allow=(capi.ERR_CAPACITY,))
        return self._result(res)
