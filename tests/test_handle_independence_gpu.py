"""GPU: a stage's handle gives the same result whatever other handles exist.

A kernel's dynamic shared-memory limit (cudaFuncAttributeMaxDynamicSharedMemorySize) belongs to the function on the
device, not to a handle: a create that set it to its own size would break every live handle that needs more.  These
tests create handles of different sizes next to each other, run them again after the others exist, and require every
result to be bit-identical to the handle's first run:

* spectrum handles of 8 ... 12289 bins, every larger one re-run after a smaller one was created;
* two pipelines whose spectrum stages differ in size, the larger one submitted eagerly and as a graph replay;
* CAF handles for every default range and Doppler instance, Wiener-Hopf handles for every solve kernel, detection
  handles of 21 and 16384 delay bins and the spectrum handles, all alive at once and re-run in reverse order, each on
  its own stream, with one synchronise at the end;
* b200dd_wh_process_device_f64, in place and out of place, against the host path and the oracle.
"""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import edge_cases as E
from blah2_b200 import capi
from blah2_b200.process import Ambiguity, Pipeline, SpectrumAnalyser, WienerHopf, _DetHandle
from blah2_b200.scene import make_scene, random_iq, Target
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

SPECTRUM_BINS = [8, 2000, 3072, 3073, 10000, 12288, 12289]
SPECTRUM_DEC = 3


def _spectrum(ns):
    n = ns * SPECTRUM_DEC
    sa = SpectrumAnalyser(n, n / (SPECTRUM_DEC + 0.5))
    assert sa.nSpectrum == ns
    return sa


def _spectrum_input(ns):
    x, _ = random_iq(ns * SPECTRUM_DEC, seed=ns)
    return torch.from_numpy(x.astype(np.complex64)).cuda()


def _spectrum_run(sa, dx, out, stream=None):
    """b200dd_spectrum_process_device into `out`: (return code, last error)."""
    lib = capi.load()
    rc = lib.b200dd_spectrum_process_device(sa._h, capi.ptr(dx), int(dx.numel()), capi.ptr(out),
                                            capi.ptr(stream) if stream else None)
    return rc, (capi.last_error() if rc != capi.OK else "")


def _spectrum_once(sa, dx):
    out = torch.empty(sa.nSpectrum, dtype=torch.complex128, device="cuda")
    rc, msg = _spectrum_run(sa, dx, out)
    torch.cuda.synchronize()
    assert rc == capi.OK, (sa.nSpectrum, rc, msg)
    return out.cpu().numpy()


@pytest.mark.parametrize("a,b", [(a, b) for a, b in itertools.permutations(SPECTRUM_BINS, 2) if a > b],
                         ids=lambda v: str(v))
def test_spectrum_handle_unchanged_by_a_smaller_handle(a, b):
    dxa, dxb = _spectrum_input(a), _spectrum_input(b)
    ha = _spectrum(a)
    first_a = _spectrum_once(ha, dxa)
    hb = _spectrum(b)
    again_a = torch.empty(a, dtype=torch.complex128, device="cuda")
    rc, msg = _spectrum_run(ha, dxa, again_a)
    torch.cuda.synchronize()
    assert rc == capi.OK, f"{a} bins after a {b}-bin handle was created: rc {rc}: {msg}"
    assert np.array_equal(again_a.cpu().numpy(), first_a)
    first_b = _spectrum_once(hb, dxb)
    fresh_b = _spectrum(b)
    assert np.array_equal(_spectrum_once(fresh_b, dxb), first_b)
    ref, _ = O.spectrum_process(dxa.cpu().numpy().astype(np.complex128), ha.nfft, ha.nfft / (SPECTRUM_DEC + 0.5))
    assert np.max(np.abs(first_a - ref)) < 1e-11 * np.max(np.abs(ref))


# ----------------------------------------------------------------------------------------------------- pipelines
METRICS = (0.0, -1.005, 1e21)


@pytest.mark.parametrize("path", ["eager", "replay"])
def test_pipeline_spectrum_unchanged_by_a_smaller_pipeline(path):
    fs, n = 2000000, 200000
    geom = (-5, 60, -500, 500, fs, n)
    sc = make_scene(n, fs, seed=23, targets=[Target(17, 300.0, -25.0)])
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    big = Pipeline(*geom, roundHamming=True, spectrum_bandwidth=10000.0)
    big.enable_iqdata_json(*METRICS)
    assert big.n_spectrum == 10000
    shape = (big.geometry.n_doppler_bins, big.geometry.n_delay_bins)
    dmap = {p: torch.zeros(shape, dtype=torch.complex64, device="cuda") for p in ("eager", "replay")}
    ts = 1700000000000

    def cpi(p):
        big.submit_device(dx, dy, dmap[p])
        big.fetch()
        return big.fetch_spectrum(), big.fetch_iqdata_json(ts), dmap[p].cpu().numpy().copy()

    before = cpi("eager")
    big.prepare_device(dx, dy, dmap["replay"])   # records the graph (and runs one CPI)
    big.fetch()
    small = Pipeline(*geom, roundHamming=True, spectrum_bandwidth=2000.0)
    assert small.n_spectrum == 2000
    after = cpi(path)
    assert np.array_equal(after[0], before[0])
    assert after[1] == before[1]
    assert np.array_equal(after[2], before[2])
    small.submit_device(dx, dy)
    small.fetch()
    ref, _ = O.spectrum_process(sc.x.astype(np.complex64).astype(np.complex128), n, 2000.0)
    assert np.max(np.abs(small.fetch_spectrum() - ref)) < 1e-11 * np.max(np.abs(ref))
    small.close()
    big.close()


# -------------------------------------------------------------------------------------------- every stage at once
def _caf_rows():
    """One CAF_ROWS geometry per default range instance and per Doppler instance."""
    rows, seen_m, seen_m2 = [], set(), set()
    for r in E.CAF_ROWS:
        if r["M"] not in seen_m or r["M2"] not in seen_m2:
            rows.append(r)
            seen_m.add(r["M"])
            seen_m2.add(r["M2"])
    return rows


# one (delayMin, delayMax) per solve kernel the tap count delayMax - delayMin selects
WH_TAPS = [(-10, 60), (0, 460), (-20, 700), (0, 1000), (-5, 1500), (0, 3000)]


def _solve_kernel(taps):
    """wh.cu wh_plan: 0 split (<= 448 taps), 1 short<512>, 2 short<1024>, 3 sweep<1>, 4 sweep<2>, 5 long."""
    return sum(taps > t for t in (448, 480, 992, 1024, 2048))


WH_N = 40000


class _Caf:
    def __init__(self, row):
        self.row = row
        self.h = Ambiguity(*row["geom"])
        g = self.h.geometry
        assert (g.range_fft_len, g.doppler_fft_len) == (row["M"], row["M2"])
        x, y = random_iq(g.n_used, seed=row["n_dop"] + row["n_del"])
        self.x, self.y = x.astype(np.complex64), y.astype(np.complex64)
        self.dx, self.dy = torch.from_numpy(self.x).cuda(), torch.from_numpy(self.y).cuda()
        self.shape = (g.n_doppler_bins, g.n_delay_bins)

    def launch(self, stream=None):
        out = torch.empty(self.shape, dtype=torch.complex64, device="cuda")
        self.h.process_device(self.dx, self.dy, out, stream=stream)
        return out

    def result(self, out):
        return out.cpu().numpy()

    def check_oracle(self, res, relerr):
        geom = self.row["geom"]
        ref, _, _ = O.ambiguity_process(self.x.astype(np.complex128), self.y.astype(np.complex128),
                                        O.ambiguity_geometry(*geom))
        e = relerr(res.astype(np.complex128), ref)
        assert e[0] < 1e-5 and e[1] < 1e-5, (E.row_id(self.row), e)


class _Wh:
    def __init__(self, taps):
        self.taps = taps
        self.h = WienerHopf(taps[0], taps[1], WH_N)
        sc = make_scene(WH_N, 2e6, seed=taps[1], targets=[Target(25, 300.0, -40.0)])
        self.x, self.y = sc.x.astype(np.complex64), sc.y.astype(np.complex64)
        self.dx, self.dy = torch.from_numpy(self.x).cuda(), torch.from_numpy(self.y).cuda()

    def launch(self, stream=None):
        out = torch.empty(WH_N, dtype=torch.complex64, device="cuda")
        self.h.process_device(self.dx, self.dy, out, stream=stream)
        return out

    def result(self, out):
        assert self.h.last_status(), self.taps
        return out.cpu().numpy()

    def check_oracle(self, res, relerr):
        ok, ref = O.wienerhopf_process(self.x.astype(np.complex128), self.y.astype(np.complex128), *self.taps)
        assert ok
        assert relerr(res.astype(np.complex128), ref)[0] < 1e-6, self.taps


class _Det:
    PARAMS = dict(pfa=1e-3, nGuard=2, nTrain=6, minDelay=-128, minDoppler=0.0)

    def __init__(self, n_dop, n_del):
        p = self.PARAMS
        self.n_dop, self.n_del = n_dop, n_del
        self.h = _DetHandle(pfa=p["pfa"], nGuard=p["nGuard"], nTrain=p["nTrain"], minDelay=p["minDelay"],
                            minDoppler=p["minDoppler"], nCentroidDelay=3, nCentroidDoppler=3, resolutionDoppler=0.5,
                            max_doppler_bins=n_dop, max_delay_bins=n_del)
        rng = np.random.default_rng(n_del)
        self.m = ((rng.standard_normal((n_dop, n_del)) + 1j * rng.standard_normal((n_dop, n_del))) * 30.0).astype(np.complex64)
        self.dm = torch.from_numpy(self.m).cuda()
        self.delay = np.ascontiguousarray(np.arange(n_del, dtype=np.int32) - 10)
        self.doppler = np.ascontiguousarray((np.arange(n_dop, dtype=np.float64) - n_dop // 2) * 0.5)

    def launch(self, stream=None):
        lib = self.h._lib
        capi.check(lib.b200dd_det_chain_device_async(self.h._h, capi.DET_INTERPOLATE, capi.ptr(self.dm), self.n_dop,
                                                     self.n_del, capi.ptr(self.delay), capi.ptr(self.doppler),
                                                     capi.ptr(stream) if stream else None))
        return stream

    def result(self, stream):
        lib = self.h._lib
        metrics = np.empty(2)
        out = [np.empty(self.h.cap) for _ in range(3)]
        n = C.c_uint32()
        capi.check(lib.b200dd_det_chain_fetch(self.h._h, capi.ptr(metrics), *(capi.ptr(o) for o in out), self.h.cap,
                                              C.byref(n), capi.ptr(stream) if stream else None))
        return np.concatenate([metrics] + [o[:n.value] for o in out])

    def check_oracle(self, res, relerr):
        p = self.PARAMS
        noise = O.set_metrics(self.m.astype(np.complex128))[0]
        assert abs(res[0] - noise) < 1e-6
        cfar = E.cfar_1d(self.m, self.delay, self.doppler, res[0], p["pfa"], p["nGuard"], p["nTrain"], p["minDelay"],
                         p["minDoppler"])
        cen = E.centroid(*cfar, 3, 3, 0.5)
        ref = O.interpolate(*cen, self.m.astype(np.complex128), self.delay, self.doppler, res[0], True, True)
        k = ref[0].shape[0]
        assert k > 0 and res.shape[0] == 2 + 3 * k, (self.n_del, k, res.shape)
        got = res[2:].reshape(3, k)
        for a, b, tol in zip(got, ref, (1e-9, 1e-9, 1e-9)):
            assert np.array_equal(np.isnan(a), np.isnan(b))
            ok = ~np.isnan(b)
            assert np.all(np.abs(a[ok] - b[ok]) <= tol)


class _Spec:
    def __init__(self, ns):
        self.h = _spectrum(ns)
        self.dx = _spectrum_input(ns)

    def launch(self, stream=None):
        out = torch.empty(self.h.nSpectrum, dtype=torch.complex128, device="cuda")
        self.h.process_device(self.dx, d_spectrum=out, stream=stream)
        return out

    def result(self, out):
        return out.cpu().numpy()

    def check_oracle(self, res, relerr):
        ref, _ = O.spectrum_process(self.dx.cpu().numpy().astype(np.complex128), self.h.nfft,
                                    self.h.nfft / (SPECTRUM_DEC + 0.5))
        assert relerr(res, ref)[0] < 1e-11


def test_every_stage_unchanged_by_the_other_live_handles(relerr):
    makers = [lambda r=r: _Caf(r) for r in _caf_rows()]
    makers += [lambda t=t: _Wh(t) for t in WH_TAPS]
    makers += [lambda d=d: _Det(*d) for d in ((31, 21), (31, 16384))]
    makers += [lambda ns=ns: _Spec(ns) for ns in SPECTRUM_BINS]
    stages, first = [], []
    for make in makers:        # each runs right after its creation
        s = make()
        out = s.launch()
        torch.cuda.synchronize()
        first.append(s.result(out))
        stages.append(s)
    ms = {int(s.h.geometry.range_fft_len) for s in stages if isinstance(s, _Caf)}
    m2s = {int(s.h.geometry.doppler_fft_len) for s in stages if isinstance(s, _Caf)}
    assert ms == {1 << l for l in range(8, 14)} and m2s == {1 << l for l in range(8, 15)}
    assert sorted(_solve_kernel(s.h.nBins) for s in stages if isinstance(s, _Wh)) == list(range(len(WH_TAPS)))
    # all alive: again in reverse order, each on its own stream, one synchronise for all of them
    streams = [torch.cuda.Stream() for _ in stages]
    pending = [(s, s.launch(st.cuda_stream)) for s, st in zip(reversed(stages), reversed(streams))]
    torch.cuda.synchronize()
    again = {id(s): s.result(p if not isinstance(s, _Det) else st.cuda_stream)
             for (s, p), st in zip(pending, reversed(streams))}
    for s, f in zip(stages, first):
        assert np.array_equal(again[id(s)], f), type(s).__name__
        s.check_oracle(f, relerr)


# ------------------------------------------------------------------------------------ WienerHopf, FP64 device entry
@pytest.mark.parametrize("taps", [(-10, 60), (0, 410)])
def test_wh_process_device_f64_in_and_out_of_place(taps, relerr):
    n = 20011
    x, y = random_iq(n, seed=taps[1])
    wh = WienerHopf(taps[0], taps[1], n)
    ok, host = wh.process(x, y)
    assert ok
    lib = capi.load()
    dx = torch.from_numpy(x).cuda()
    for inplace in (False, True):
        dy = torch.from_numpy(y).cuda()
        out = dy if inplace else torch.full_like(dy, complex(np.nan, np.nan))
        torch.cuda.synchronize()
        capi.check(lib.b200dd_wh_process_device_f64(wh._h, capi.ptr(dx), capi.ptr(dy), capi.ptr(out), None))
        assert wh.last_status()
        got = out.cpu().numpy()
        assert np.array_equal(got, host), inplace
        if not inplace:
            assert np.array_equal(dy.cpu().numpy(), y)    # the input is left alone
    ok_ref, ref = O.wienerhopf_process(x, y, *taps)
    assert ok_ref and relerr(host, ref)[0] < 1e-9
