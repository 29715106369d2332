"""The detection tail on the device, bit for bit, on the boundary cases of tests/det_cases.py.

Expected lists come from the restatement in det_cases fed with the device's own per-cell values: the dB value of
every cell is the map document's cell_db (b200dd_mapjson_debug_cell_values), and |z z| is hypot of the separately
rounded complex square taken by torch.hypot on CUDA doubles, the same libm the kernels call.  No libm difference is
left, so every list must match exactly, NaN where NaN.  Two libm assumptions the tie cases rest on are checked on the
device once per case set: hypot(a, 0) == |a|, and log10 of the plateau pair keeps the pair a plateau; a case whose
assumption fails is reported and still compared bit for bit.

Map::set_metrics is checked against a rigorous bound around the exact mean of the device's cell values, built from
the reduction's shape, and its maxPower bit for bit.
"""
import ctypes as C
import math
import os
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import det_cases as D  # noqa: E402

from blah2_b200 import capi  # noqa: E402
from blah2_b200.process import Detection, Map, MapJson, Pipeline, _DetHandle  # noqa: E402
from oracle import refpath  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

CFAR_CASES = D.cfar_cases()
FLAGS = [(True, True), (True, False), (False, True), (False, False)]
STAGES = (capi.DET_CFAR, capi.DET_CENTROID, capi.DET_INTERPOLATE)


@pytest.fixture(scope="module", autouse=True)
def _report_runtime():
    t0 = time.perf_counter()
    yield
    print(f"\ntest_det_exact_gpu: {time.perf_counter() - t0:.1f} s")


def _dev_hypot(a, b):
    return torch.hypot(torch.from_numpy(np.ascontiguousarray(a)).cuda(),
                       torch.from_numpy(np.ascontiguousarray(b)).cuda()).cpu().numpy()


def dev_sq(m):
    return D.sq_values(np.asarray(m, np.complex128), hypot=_dev_hypot)


def dev_db(t, delay, doppler, noise):
    """cell_db of every cell of the device map t (complex64 or complex128) at noise."""
    mj = MapJson(delay, doppler, 2000000)
    try:
        return mj.cell_values(t, noise)
    finally:
        mj.close()


def _handle(p, shape):
    return _DetHandle(pfa=p["pfa"], nGuard=p["nGuard"], nTrain=p["nTrain"], minDelay=p["minDelay"],
                      minDoppler=p["minDoppler"], nCentroidDelay=p["nCentroidDelay"],
                      nCentroidDoppler=p["nCentroidDoppler"], resolutionDoppler=p["resolutionDoppler"],
                      doDelay=p["doDelay"], doDoppler=p["doDoppler"], max_doppler_bins=shape[0],
                      max_delay_bins=shape[1])


def _dev_log10(m):
    return torch.log10(torch.from_numpy(np.abs(m)).cuda()).cpu().numpy()


def _lists(det):
    return det.delay, det.doppler, det.snr


def _chain_async(h, stage, t, delay, doppler):
    """b200dd_det_chain_device_async + b200dd_det_chain_fetch: ((noisePower, maxPower), list)."""
    delay = np.ascontiguousarray(delay, dtype=np.int32)
    doppler = np.ascontiguousarray(doppler, dtype=np.float64)
    capi.check(h._lib.b200dd_det_chain_device_async(h._h, stage, capi.ptr(t), t.shape[0], t.shape[1],
                                                    capi.ptr(delay), capi.ptr(doppler), None))
    met = np.empty(2)
    od, of, os_ = h._bufs(h.cap)
    n = C.c_uint32()
    capi.check(h._lib.b200dd_det_chain_fetch(h._h, capi.ptr(met), capi.ptr(od), capi.ptr(of), capi.ptr(os_), h.cap,
                                             C.byref(n), None))
    k = n.value
    return (float(met[0]), float(met[1])), (od[:k].copy(), of[:k].copy(), os_[:k].copy())


def _assert_same(got, want, what):
    assert D.same(got, want), (what, len(got[0]), len(want[0]))


def test_device_hypot_of_a_real_cell_is_its_magnitude():
    """The tie cases take |z| = |x| and |z z| = x^2 for a real cell x: CUDA's hypot(a, 0) must return |a|."""
    vals = np.concatenate([c["map"].real.ravel() for c in CFAR_CASES])
    vals = np.concatenate([vals, vals * vals, -vals])
    assert np.array_equal(_dev_hypot(vals, np.zeros_like(vals)), np.abs(vals))


@pytest.mark.parametrize("case", CFAR_CASES, ids=lambda c: c["name"])
def test_cfar_cases_on_every_map_entry_point(case):
    p, m = case["params"], case["map"]
    h = _handle(p, m.shape)
    t64 = torch.from_numpy(m).cuda()
    sq = dev_sq(m)
    try:
        db = dev_db(t64, case["delay"], case["doppler"], D.NOISE)
        for stage in STAGES:  # double map
            got = _lists(h.process_map(Map(m, case["delay"], case["doppler"], D.NOISE), stage))
            _assert_same(got, D.chain(sq, db, case["delay"], case["doppler"], p, stage), ("host", stage))
        if not case["f32"]:
            return
        t32 = torch.from_numpy(m.astype(np.complex64)).cuda()
        db32 = dev_db(t32, case["delay"], case["doppler"], D.NOISE)
        assert np.array_equal(db32, db)
        for stage in STAGES:  # float map, given noise
            got = _lists(h.process_device_map(t32, m.shape[0], m.shape[1], case["delay"], case["doppler"], D.NOISE,
                                              stage))
            _assert_same(got, D.chain(sq, db, case["delay"], case["doppler"], p, stage), ("device", stage))
        for stage in STAGES:  # device-resident chain: set_metrics' noise, the fused tail kernel
            (noise, _), got = _chain_async(h, stage, t32, case["delay"], case["doppler"])
            dbn = dev_db(t32, case["delay"], case["doppler"], noise)
            _assert_same(got, D.chain(sq, dbn, case["delay"], case["doppler"], p, stage), ("chain", stage))
    finally:
        h.close()


@pytest.mark.parametrize("n_det", [1023, 1024, 1025, 2049])
def test_long_lists_through_the_fused_tail(n_det):
    """Lists across the one-CTA tail kernel's 1024-thread compaction, through the device chain and the separate
    kernels."""
    m, delay, doppler = D.spike_map(n_det)
    p = D.det_params(nGuard=1, nTrain=2, nCentroidDelay=2, nCentroidDoppler=2, resolutionDoppler=10.0)
    h = _handle(p, m.shape)
    try:
        t32 = torch.from_numpy(m.astype(np.complex64)).cuda()
        sq = dev_sq(m)
        assert len(D.cfar(sq, sq, delay, doppler, p["pfa"], 1, 2, p["minDelay"], 0.0)[0]) == n_det
        for stage in STAGES:
            (noise, _), got = _chain_async(h, stage, t32, delay, doppler)
            _assert_same(got, D.chain(sq, dev_db(t32, delay, doppler, noise), delay, doppler, p, stage), stage)
            got = _lists(h.process_device_map(t32, m.shape[0], m.shape[1], delay, doppler, noise, stage))
            _assert_same(got, D.chain(sq, dev_db(t32, delay, doppler, noise), delay, doppler, p, stage), stage)
    finally:
        h.close()


def test_centroid_cases_on_centroid_host():
    P = D.CENTROID_PARAMS
    p = D.det_params(nCentroidDelay=P["nDelay"], nCentroidDoppler=P["nDoppler"], resolutionDoppler=P["res"])
    h = _handle(p, (64, 64))
    try:
        for name, d, f, s in D.centroid_cases():
            got = _lists(h.centroid(Detection(d, f, s)))
            _assert_same(got, D.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"]), name)
            if refpath.available():
                _assert_same(got, refpath.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"]), name)
    finally:
        h.close()


def _device_plateau_pair():
    """The first plateau pair that stays one under CUDA's log10 (the libm guard), and the candidates it dropped."""
    dropped = []
    for a, b in D.plateau_pairs():
        L = torch.log10(torch.tensor([a, b], dtype=torch.float64, device="cuda")).cpu().numpy()
        if L[1] < L[0] and 10.0 * L[0] == 10.0 * L[1] and D.fma(L[1], 10.0, -D.NOISE) < D.fma(L[0], 10.0, -D.NOISE):
            return (a, b), dropped
        dropped.append((a, b))
    return None, dropped


@pytest.mark.parametrize("flags", FLAGS)
def test_interpolate_case_on_interpolate_host(flags):
    pair, dropped = _device_plateau_pair()
    if dropped:
        print(f"plateau pairs dropped, not plateaus under CUDA's log10: {dropped}")
    assert pair is not None, "no plateau pair survives CUDA's log10"
    case = D.interp_case(pair=pair)
    p = D.det_params(doDelay=flags[0], doDoppler=flags[1])
    h = _handle(p, case["map"].shape)
    try:
        t64 = torch.from_numpy(case["map"]).cuda()
        db = dev_db(t64, case["delay"], case["doppler"], case["noise"])
        got = _lists(h.interpolate(Detection(*case["list"]), Map(case["map"], case["delay"], case["doppler"],
                                                                case["noise"])))
        want = D.interpolate(*case["list"], db, case["delay"], case["doppler"], *flags)
        _assert_same(got, want[:3], flags)
        if flags[0] and not flags[1]:
            assert np.isnan(got[2]).any()
        if flags != (False, False):  # the plateau pair's detection stays, where the fused dB value dropped it
            fused = D.interpolate(*case["list"], D.db_values(_dev_log10(case["map"]), case["noise"], fused=True),
                                  case["delay"], case["doppler"], *flags)
            assert len(fused[0]) < len(got[0])
    finally:
        h.close()


def _pipeline_case():
    from blah2_b200.scene import Target, make_scene

    fs, n = 200000, 40000
    geom = (-5, 60, -500, 500, fs, n)
    det = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
    sc = make_scene(n, fs, seed=11, targets=[Target(17, 300.0, -25.0), Target(41, -200.0, -28.0)])
    p = D.det_params(pfa=det["pfa"], nGuard=det["nGuard"], nTrain=det["nTrain"], minDelay=det["minDelay"],
                     minDoppler=det["minDoppler"], nCentroidDelay=det["nCentroid"], nCentroidDoppler=det["nCentroid"],
                     resolutionDoppler=1.0 / (float(n) / float(fs)))
    return geom, det, sc, p


def _check_pipeline_cpi(pipe, p, m, noise, max_power, det):
    t = torch.from_numpy(np.ascontiguousarray(m)).cuda()
    want = D.chain(dev_sq(m), dev_db(t, pipe.delay, pipe.doppler, noise), pipe.delay, pipe.doppler, p)
    _assert_same(_lists(det), want, "pipeline")
    _check_metrics(dev_db(t, pipe.delay, pipe.doppler, 0.0), noise, max_power, grid_cells=m.size)
    return len(want[0])


def test_pipeline_detections_are_the_restatement_on_its_own_map():
    geom, det, sc, p = _pipeline_case()
    pipe = Pipeline(*geom, roundHamming=True, clutter=(-5, 30), detection=det, device=0)
    try:
        out = pipe.process(sc.x, sc.y)
        assert _check_pipeline_cpi(pipe, p, out["map"], out["noisePower"], out["maxPower"], out["detections"]) >= 2
        dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
        dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
        dmap = torch.empty((pipe.geometry.n_doppler_bins, pipe.geometry.n_delay_bins), dtype=torch.complex64,
                           device="cuda")
        pipe.prepare_device(dx, dy, dmap)  # every submit of this triple replays the recorded graph
        for _ in range(2):
            pipe.submit_device(dx, dy, dmap)
            r = pipe.fetch()
            m = dmap.cpu().numpy().astype(np.complex128)
            _check_pipeline_cpi(pipe, p, m, r["noisePower"], r["maxPower"], r["detections"])
    finally:
        pipe.close()


# ---------------------------------------------------------------------------------------------- set_metrics
def _gamma(k):
    u = 2.0 ** -53
    return k * u / (1 - k * u)


def _exact_sum(v):
    """(sum, err): the exact sum of v rounded per chunk by math.fsum, and a bound on what that rounding lost."""
    parts = [math.fsum(c.tolist()) for c in np.array_split(v, max(1, v.size // (1 << 20)))]
    return math.fsum(parts), sum(math.ulp(x) for x in parts) / 2 + math.ulp(math.fsum(parts))


def _check_metrics(v, noise, max_power, grid_cells):
    """v: every cell's 10 log10|z| as the device computes it.  noisePower is their sum over a grid-stride loop of
    ceil(cells / (grid 256)) terms per thread, 5 shuffle levels, 8 warp partials, ceil(grid / 256) partials per thread
    of the final block and an 8-level tree, then one division: within gamma_depth sum|v| / cells of the exact mean."""
    v = np.asarray(v, dtype=np.float64).ravel()
    cells = v.size
    assert cells == grid_cells
    finite = v[np.isfinite(v)]
    vmax = max(0.0, float(np.max(v[~np.isnan(v)]))) if np.any(~np.isnan(v)) else 0.0
    if np.isnan(v).any():
        assert math.isnan(noise) and math.isnan(max_power)
        return
    if np.isneginf(v).any():
        assert noise == -math.inf and max_power == vmax - noise
        return
    assert finite.size == cells
    grid = min((cells + 255) // 256, 592)
    depth = -(-cells // (grid * 256)) + 5 + 8 + -(-grid // 256) + 8
    s, err = _exact_sum(v)
    mean = s / cells
    abs_sum = float(np.sum(np.abs(v))) * (1 + 1e-9)  # an upper bound on sum|v| is all the bound needs
    bound = _gamma(depth) * abs_sum / cells + err / cells + math.ulp(abs(mean)) * 2
    assert abs(noise - mean) <= bound, (noise, mean, bound)
    assert max_power == vmax - noise


def _torch_cell_db0(t):
    """10 log10|z| per cell in separately rounded CUDA double operations (torch's hypot and log10 are CUDA's)."""
    z = torch.view_as_real(t).double()
    return torch.mul(torch.log10(torch.hypot(z[..., 0], z[..., 1])), 10.0)


@pytest.mark.parametrize("shape", [(1, 1), (1, 255), (7, 37), (1, 592 * 256 - 1), (1, 592 * 256 + 1),
                                   (8191, 16384)])
def test_set_metrics_within_the_reduction_bound(shape):
    g = torch.Generator("cuda").manual_seed(shape[1])
    t = torch.complex(torch.randn(shape, device="cuda", generator=g), torch.randn(shape, device="cuda", generator=g)) * 30.0
    h = _DetHandle(max_doppler_bins=min(shape[0], 8192), max_delay_bins=min(shape[1], 16384))
    try:
        v = _torch_cell_db0(t)
        if t.numel() < 1 << 22:  # torch's values are the map document's
            assert np.array_equal(v.cpu().numpy(), dev_db(t, np.arange(shape[1]), np.arange(shape[0]) * 1.0, 0.0))
        noise, mx = h.set_metrics_device(t, shape[0], shape[1])
        torch.cuda.synchronize()
        _check_metrics(v.cpu().numpy(), noise, mx, t.numel())
        if shape[1] <= 16384:
            delay, doppler = np.arange(shape[1], dtype=np.int32), np.arange(shape[0], dtype=np.float64)
            (n2, m2), _ = _chain_async(h, 0, t, delay, doppler)
            assert (n2, m2) == (noise, mx)
    finally:
        h.close()


@pytest.mark.parametrize("kind", ["zero_cell", "all_below_one", "nan_cell"])
def test_set_metrics_special_maps(kind):
    shape = (7, 37)
    m = (np.random.default_rng(3).uniform(0.1, 0.9, shape) + 0j).astype(np.complex64)
    if kind == "zero_cell":
        m[3, 5] = 0
    if kind == "nan_cell":
        m[6, 36] = complex(np.nan, 0)
    t = torch.from_numpy(m).cuda()
    h = _DetHandle(max_doppler_bins=shape[0], max_delay_bins=shape[1])
    try:
        v = dev_db(t, np.arange(shape[1]), np.arange(shape[0]) * 1.0, 0.0)
        noise, mx = h.set_metrics_device(t, *shape)
        _check_metrics(v, noise, mx, t.numel())
        if kind == "all_below_one":
            assert mx == -noise  # the running max starts at 0 (Map.cpp:193)
        (n2, m2), _ = _chain_async(h, 0, t, np.arange(shape[1], dtype=np.int32), np.arange(shape[0], dtype=np.float64))
        assert np.array_equal([n2, m2], [noise, mx], equal_nan=True)
    finally:
        h.close()
