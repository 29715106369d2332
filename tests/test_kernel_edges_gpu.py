"""GPU: the default kernel instances at their plan boundaries, on misaligned guard-banded buffers, and the detection
kernels on large maps.

* Every row of tests/edge_cases.CAF_ROWS (each default (range M, Doppler M2) instance, both sides of every boundary)
  against the oracle.
* The TMA-staged default kernels (caf_range_dit_kernel, the float2 Wiener-Hopf kernels) on inputs that start on a
  16-byte or only an 8-byte boundary and end at the array's end, with NaN guards around every buffer: a read outside
  an input brings a NaN into the result, a write outside an output changes a guard.
* CFAR / Centroid / Interpolate on maps up to 8191 rows and 16384 delay bins with thousands of detections, and the
  list-capacity error paths, against the vectorised restatements of tests/edge_cases.py.
"""
import ctypes as C
import itertools

import numpy as np
import pytest

import edge_cases as E
from blah2_b200 import capi
from blah2_b200.process import Ambiguity, Pipeline, WienerHopf, WienerHopfChunk, _DetHandle
from blah2_b200.scene import make_scene, random_iq, Target
from guarded import Guarded
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _c64(a):
    return np.asarray(a).astype(np.complex64)


def _sync():
    import torch
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ B: CAF plan edges
@pytest.mark.parametrize("row", E.CAF_ROWS, ids=E.row_id)
def test_default_caf_kernels_match_the_oracle_at_every_plan_edge(row, relerr):
    geom = row["geom"]
    x, y = random_iq(geom[5], seed=row["n_dop"] + row["n_del"])
    x, y = _c64(x).astype(np.complex128), _c64(y).astype(np.complex128)
    amb = Ambiguity(*geom)
    g = amb.geometry
    assert (g.range_fft_len, g.doppler_fft_len, g.n_delay_bins, g.n_doppler_bins) == (row["M"], row["M2"], row["n_del"], row["n_dop"])
    m = amb.process(x, y).data
    R = amb.debug_range_matrix()
    og = O.ambiguity_geometry(*geom)
    Rref = O.range_matrix(O.ambiguity_prerotate(x, og), y, og)
    e_r = relerr(R, Rref)
    e = relerr(m, O.doppler_transform(Rref, og))
    assert e_r[0] < TOL and e_r[1] < TOL, f"range matrix {e_r}"
    assert e[0] < TOL and e[1] < TOL, f"map {e}"
    assert np.array_equal(amb.process(x, y).data, m)


# ------------------------------------------------------------------------- C: CAF on misaligned, guarded buffers
# one geometry per default range instance; delayMin < 0, = 0 and > 0; symmetric Doppler windows (an asymmetric one
# reads a pre-rotated, aligned copy of x)
MISALIGNED_CAF = [
    ((-3, 60, -200, 200, 100000, 100000, True), 256),
    ((0, 200, -100, 100, 200000, 400000, True), 512),
    ((5, 520, -60, 60, 100000, 300000, True), 1024),
    ((0, 900, -30, 30, 100000, 400000, True), 2048),
    ((7, 2000, -20, 20, 100000, 600000, True), 4096),
    ((-50, 3100, -15, 15, 100000, 400000, True), 8192),
]


@pytest.mark.parametrize("geom,M", MISALIGNED_CAF, ids=[f"M{m}" for _, m in MISALIGNED_CAF])
def test_caf_on_misaligned_guarded_buffers(geom, M, relerr):
    amb = Ambiguity(*geom)
    g = amb.geometry
    assert g.range_fft_len == M and g.doppler_middle == 0.0
    n, cells = g.n_used, g.n_doppler_bins * g.n_delay_bins
    x, y = (_c64(v) for v in random_iq(n, seed=M))
    maps = {}
    for ox, oy in itertools.product((0, 1), repeat=2):
        bx, by, bm = Guarded(n, ox, x), Guarded(n, oy, y), Guarded(cells, 1)
        _sync()
        amb.process_device(bx.view, by.view, bm.view)
        _sync()
        assert bx.intact() and by.intact() and bm.intact(), (ox, oy)
        maps[(ox, oy)] = bm.numpy()
    base = maps[(0, 0)]
    assert np.all(np.isfinite(base))
    for k, v in maps.items():
        assert np.array_equal(v, base), f"x/y offsets {k}"
    ref, _, _ = O.ambiguity_process(x.astype(np.complex128), y.astype(np.complex128), O.ambiguity_geometry(*geom))
    e = relerr(base.reshape(ref.shape).astype(np.complex128), ref)
    assert e[0] < TOL and e[1] < TOL, e


@pytest.mark.parametrize("geom", [(-4, 200, -20, 20, 100000, 100000, True), (-5, 60, -20, 20, 100000, 100000, True)])
def test_range_stage_on_every_batch_slice_of_misaligned_buffers(geom):
    """b200dd_caf_range_device one batch at a time: with an odd nCorr the slices alternate between 16- and 8-byte
    aligned starts, and the last one ends at the end of the buffer.  Their range matrix, through
    b200dd_caf_doppler_device, must give the one-shot map bit for bit."""
    amb = Ambiguity(*geom)
    g = amb.geometry
    nc, nd, nl = g.n_corr, g.n_doppler_bins, g.n_delay_bins
    assert nc % 2 == 1
    x, y = (_c64(v) for v in random_iq(g.n_used, seed=nc))
    for ox, oy in itertools.product((0, 1), repeat=2):
        bx, by = Guarded(g.n_used, ox, x), Guarded(g.n_used, oy, y)
        full, R, tile = Guarded(nd * nl, 1), Guarded(nd * nl, 1), Guarded(nd * nl, 1)
        _sync()
        amb.process_device(bx.view, by.view, full.view)
        for b in range(nd):
            amb.range_device(bx.view[b * nc:(b + 1) * nc], by.view[b * nc:(b + 1) * nc], b, 1, R.view[b * nl:(b + 1) * nl])
        amb.doppler_device(R.view, 0, nl, tile.view)
        _sync()
        assert all(b.intact() for b in (bx, by, full, R, tile)), (ox, oy)
        assert np.all(np.isfinite(full.numpy()))
        assert np.array_equal(tile.numpy(), full.numpy()), (ox, oy)


# --------------------------------------------------------------- C: float2 clutter filter on misaligned buffers
WH_OFFSETS = [(ox, oy, oo, False) for ox, oy, oo in itertools.product((0, 1), repeat=3)] + \
             [(ox, oy, oy, True) for ox, oy in itertools.product((0, 1), repeat=2)]


def _wh_device_runs(wh, x, y):
    """WienerHopf.process_device (float2) for every (x, y, y_out) offset and in place; the results, bit-identical."""
    n = x.shape[0]
    outs = []
    for ox, oy, oo, inplace in WH_OFFSETS:
        bx, by = Guarded(n, ox, x), Guarded(n, oy, y)
        bo = by if inplace else Guarded(n, oo)
        _sync()
        wh.process_device(bx.view, by.view, bo.view)
        _sync()
        assert wh.last_status()
        assert bx.intact() and by.intact() and bo.intact(), (ox, oy, oo, inplace)
        outs.append(bo.numpy())
    assert np.all(np.isfinite(outs[0]))
    for (ox, oy, oo, inplace), o in zip(WH_OFFSETS, outs):
        assert np.array_equal(o, outs[0]), (ox, oy, oo, inplace)
    return outs[0].astype(np.complex128)


def _wh_check(wh, x, y, dm, dM, relerr):
    got = _wh_device_runs(wh, x, y)
    ok, host = wh.process(x, y)
    ok_ref, ref = O.wienerhopf_process(x.astype(np.complex128), y.astype(np.complex128), dm, dM)
    assert ok and ok_ref
    assert relerr(got, host)[0] < 1e-6 and relerr(got, ref)[0] < 1e-6, (relerr(got, host), relerr(got, ref))


@pytest.mark.parametrize("window", [(-10, 40), (0, 50), (3, 60)])
@pytest.mark.parametrize("log2m", [9, 10, 11, 12])
@pytest.mark.parametrize("stage", ["CORR", "APPLY"])
def test_filter_device_path_on_misaligned_buffers_at_every_fft_length(stage, log2m, window, relerr, monkeypatch):
    monkeypatch.setenv(f"B200DD_WH_{stage}_LOG2M", str(log2m))
    n = 20011
    dm, dM = window
    sc = make_scene(n, 2e6, seed=16 * log2m + dm + 10, targets=[Target(25, 300.0, -40.0)])
    x, y = _c64(sc.x), _c64(sc.y)
    wh = WienerHopf(dm, dM, n)
    assert (wh.plan.corr_fft_len if stage == "CORR" else wh.plan.filter_fft_len) == 1 << log2m
    _wh_check(wh, x, y, dm, dM, relerr)


@pytest.mark.parametrize("case", [(512, 0, 1), (512, -10, 438), (512, 5, 453), (600, -5, 55), (600, 7, 67)])
def test_filter_device_path_on_short_signals(case, relerr):
    """Signals barely longer than the FFT: the correlation windows wrap around the end of x and are loaded directly,
    not staged."""
    n, dm, dM = case
    x, y = (_c64(v) for v in random_iq(n, seed=n + dM))
    wh = WienerHopf(dm, dM, n)
    assert wh.plan.corr_fft_len == 512
    _wh_check(wh, x, y, dm, dM, relerr)


@pytest.mark.parametrize("case", [(120000, 0, 60, 2, 8), (200003, -3, 129, 4, 9)])
def test_chunked_filter_on_misaligned_halo_buffers(case, relerr):
    """test_wh_gpu.test_chunked_filter_emulating_several_ranks with every rank's halo-exact x_loc / y_loc and its
    output in guarded buffers at 16- and 8-byte aligned starts: bit-identical to the aligned run."""
    import torch
    from blah2_b200.shard import block_range
    n, dm, dM, world, seed = case
    sc = make_scene(n, 2e6, seed=seed, targets=[Target(25, 300.0, -40.0)])
    xg, yg = _c64(sc.x), _c64(sc.y)
    wh = WienerHopf(dm, dM, n)
    whole = torch.empty(n, dtype=torch.complex64, device="cuda")
    _sync()
    wh.process_device(torch.from_numpy(xg).cuda(), torch.from_numpy(yg).cuda(), whole)
    _sync()
    chunks = []
    for r in range(world):
        c0, nc = block_range(n, r, world)
        ch = WienerHopfChunk(dm, dM, n, c0, nc)
        xl, xr, yr = ch.halos()
        chunks.append((ch, nc, xg[np.arange(c0 - xl, c0 + nc + xr) % n], yg[np.arange(c0, c0 + nc + yr) % n]))
    results = {}
    for ox, oy, oo in [(0, 0, 0), (1, 0, 1), (0, 1, 1), (1, 1, 0)]:
        bufs = [(Guarded(xl.shape[0], ox, xl), Guarded(yl.shape[0], oy, yl), Guarded(nc, oo)) for _, nc, xl, yl in chunks]
        abs_ = [torch.zeros(2 * ch.nBins, dtype=torch.complex128, device="cuda") for ch, _, _, _ in chunks]
        _sync()
        for (ch, _, _, _), (bx, by, _), ab in zip(chunks, bufs, abs_):
            ch.corr_device(bx.view, by.view, ab)
        _sync()
        ab_sum = torch.stack(abs_).sum(0)
        for (ch, _, _, _), (bx, by, bo) in zip(chunks, bufs):
            ch.filter_device(ab_sum, bx.view, by.view, bo.view)
        _sync()
        assert all(ch.last_status() for ch, _, _, _ in chunks)
        assert all(b.intact() for t in bufs for b in t), (ox, oy, oo)
        results[(ox, oy, oo)] = (ab_sum.cpu().numpy(), np.concatenate([bo.numpy() for _, _, bo in bufs]))
    ab0, y0 = results[(0, 0, 0)]
    assert np.all(np.isfinite(y0))
    for k, (ab, yk) in results.items():
        assert np.array_equal(ab, ab0) and np.array_equal(yk, y0), k
    assert relerr(y0, whole.cpu().numpy())[0] < 1e-6


def test_pipeline_device_path_on_misaligned_buffers():
    import torch
    geom = (-10, 120, -300, 300, 2000000, 400000, True)
    det = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
    sc = make_scene(geom[5], geom[4], seed=31, targets=[Target(37, 110.0, -40.0), Target(92, -205.0, -45.0)])
    x, y = _c64(sc.x), _c64(sc.y)
    pipe = Pipeline(*geom[:6], roundHamming=True, clutter=(-10, 60), detection=det)
    g = pipe.geometry
    n, cells = geom[5], g.n_doppler_bins * g.n_delay_bins
    runs = {}
    for ox, oy in [(0, 0), (1, 0), (0, 1), (1, 1)]:
        bx, by, bm = Guarded(n, ox, x), Guarded(n, oy, y), Guarded(cells, 1 - (ox & oy))
        _sync()
        pipe.submit_device(bx.view, by.view, bm.view)
        r = pipe.fetch()
        _sync()
        assert not r["skipped"] and bx.intact() and by.intact() and bm.intact(), (ox, oy)
        d = r["detections"]
        runs[(ox, oy)] = (bm.numpy(), d.delay, d.doppler, d.snr, r["noisePower"])
    base = runs[(0, 0)]
    assert np.all(np.isfinite(base[0])) and base[1].shape[0] >= 2
    for k, v in runs.items():
        assert all(np.array_equal(a, b) for a, b in zip(v, base)), k
    ref = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    _sync()
    pipe.submit_device(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), ref)
    pipe.fetch()
    _sync()
    assert np.array_equal(ref.cpu().numpy().reshape(-1), base[0])


# ----------------------------------------------------------------------------------- D: detection on large maps
def _axes(n_dop, n_del, res=0.5):
    delay = np.arange(n_del, dtype=np.int32) - 10
    doppler = (np.arange(n_dop, dtype=np.float64) - n_dop // 2) * res
    return delay, doppler


def _spike_map(n_dop, n_del, n_spikes, seed, floor=1.0):
    """A constant floor and spikes on cells two apart in both directions (even row, even column).  With nGuard = 0,
    nTrain = 1 and pfa = 1e-3 a spike is detected when S^2 > 61 b^2 (999 b^2 where one training cell is missing) and
    a floor cell never is: every CFAR decision is exact by construction, and every spike is a local maximum."""
    rng = np.random.default_rng(seed)
    m = np.full((n_dop, n_del), floor, dtype=np.complex64)
    er, ec = (n_dop + 1) // 2, (n_del + 1) // 2
    pick = rng.choice(er * ec, size=min(n_spikes, er * ec), replace=False)
    r, c = 2 * (pick // ec), 2 * (pick % ec)
    m[r, c] = (rng.uniform(40.0, 80.0, r.shape[0]) * np.exp(2j * np.pi * rng.uniform(size=r.shape[0]))).astype(np.complex64)
    return m


def _noise_map(n_dop, n_del, seed):
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal((n_dop, n_del)) + 1j * rng.standard_normal((n_dop, n_del))) * 30.0).astype(np.complex64)


SPIKES = dict(pfa=1e-3, nGuard=0, nTrain=1, minDelay=-128, minDoppler=0.0)
NOISE = dict(pfa=1e-3, nGuard=2, nTrain=6, minDelay=-128, minDoppler=0.0)

LARGE_MAPS = [
    ("spikes", 31, 16384, 1), ("spikes", 2049, 300, 3), ("spikes", 8191, 21, 3), ("spikes", 512, 1025, 1),
    ("noise", 31, 16384, 3), ("noise", 2049, 300, 3), ("noise", 8191, 21, 3),
]


def _reference(m, delay, doppler, noise, params, n_centroid, res):
    cfar = E.cfar_1d(m, delay, doppler, noise, params["pfa"], params["nGuard"], params["nTrain"], params["minDelay"],
                     params["minDoppler"])
    cen = E.centroid(*cfar, n_centroid, n_centroid, res)
    return cfar, cen, O.interpolate(*cen, m.astype(np.complex128), delay, doppler, noise, True, True)


def _same(got, ref, pos_tol=0.0, snr_tol=1e-9):
    assert got[0].shape[0] == ref[0].shape[0], (got[0].shape[0], ref[0].shape[0])
    for a, b, tol in zip(got, ref, (pos_tol, pos_tol, snr_tol)):
        assert np.array_equal(np.isnan(a), np.isnan(b))
        ok = ~np.isnan(b)
        assert a[ok].shape[0] == 0 or np.max(np.abs(a[ok] - b[ok])) <= tol


def _det_handle(params, n_dop, n_del, n_centroid, res):
    return _DetHandle(pfa=params["pfa"], nGuard=params["nGuard"], nTrain=params["nTrain"], minDelay=params["minDelay"],
                      minDoppler=params["minDoppler"], nCentroidDelay=n_centroid, nCentroidDoppler=n_centroid,
                      resolutionDoppler=res, max_doppler_bins=n_dop, max_delay_bins=n_del)


def _chain(h, stage, d_map, n_dop, n_del, delay, doppler, cap):
    """b200dd_det_chain_device_async + b200dd_det_chain_fetch: (rc, n_out, metrics, (delay, doppler, snr))."""
    lib = h._lib
    delay = np.ascontiguousarray(delay, dtype=np.int32)
    doppler = np.ascontiguousarray(doppler, dtype=np.float64)
    capi.check(lib.b200dd_det_chain_device_async(h._h, stage, capi.ptr(d_map), n_dop, n_del, capi.ptr(delay),
                                                 capi.ptr(doppler), None))
    metrics = np.empty(2)
    out = [np.full(max(1, cap), -7.0) for _ in range(3)]
    n = C.c_uint32()
    rc = lib.b200dd_det_chain_fetch(h._h, capi.ptr(metrics), *(capi.ptr(o) for o in out), cap, C.byref(n), None)
    return rc, n.value, metrics, out


@pytest.mark.parametrize("kind,n_dop,n_del,n_centroid", LARGE_MAPS, ids=[f"{k}-{a}x{b}" for k, a, b, _ in LARGE_MAPS])
def test_detection_on_large_maps(kind, n_dop, n_del, n_centroid):
    import torch
    res = 0.5
    delay, doppler = _axes(n_dop, n_del, res)
    if kind == "spikes":
        m, params = _spike_map(n_dop, n_del, 3000, seed=n_dop), SPIKES
    else:
        m, params = _noise_map(n_dop, n_del, seed=n_dop), NOISE
    d_map = torch.from_numpy(m).cuda()
    h = _det_handle(params, n_dop, n_del, n_centroid, res)
    # stand-alone kernels, noise power given
    noise = 1.25
    cfar, cen, interp = _reference(m, delay, doppler, noise, params, n_centroid, res)
    if kind == "spikes":
        assert cfar[0].shape[0] == np.count_nonzero(m != 1.0)
    assert cfar[0].shape[0] > 1024 or n_dop > 1024 or n_del > 6144
    d = h.process_device_map(d_map, n_dop, n_del, delay, doppler, noise, capi.DET_CFAR)
    _same((d.delay, d.doppler, d.snr), cfar)
    d = h.process_device_map(d_map, n_dop, n_del, delay, doppler, noise, capi.DET_CENTROID)
    _same((d.delay, d.doppler, d.snr), cen)
    d = h.process_device_map(d_map, n_dop, n_del, delay, doppler, noise, capi.DET_INTERPOLATE)
    _same((d.delay, d.doppler, d.snr), interp, pos_tol=1e-9)
    # fused chain: noise power from the device's Map::set_metrics
    for stage, which in ((capi.DET_CENTROID, 1), (capi.DET_INTERPOLATE, 2)):
        rc, k, metrics, out = _chain(h, stage, d_map, n_dop, n_del, delay, doppler, h.cap)
        assert rc == capi.OK
        assert abs(metrics[0] - O.set_metrics(m.astype(np.complex128))[0]) < 1e-6
        ref = _reference(m, delay, doppler, metrics[0], params, n_centroid, res)[which]
        _same(tuple(o[:k] for o in out), ref, pos_tol=1e-9 if which == 2 else 0.0)
    h.close()


def test_interpolate_with_all_zero_neighbours_matches_the_oracle():
    """10 log10(0) = -inf on both sides of a detection: the parabola's offset is NaN, and so is the SNR the
    reference's std::max makes of it (fmax would return the CFAR SNR instead).  Compared NaN-aware."""
    import torch
    n_dop, n_del, res = 9, 40, 0.5
    delay, doppler = _axes(n_dop, n_del, res)
    m = np.full((n_dop, n_del), 1.0, dtype=np.complex64)
    m[3:6, 10:13] = 0.0
    m[4, 11] = 50.0                     # zero on all four sides
    m[6, 30] = 60.0                     # an ordinary spike
    d_map = torch.from_numpy(m).cuda()
    h = _det_handle(SPIKES, n_dop, n_del, 1, res)
    for noise in (0.0, 2.5):
        ref = _reference(m, delay, doppler, noise, SPIKES, 1, res)[2]
        assert ref[0].shape[0] == 2 and np.isnan(ref[0]).sum() == 1
        d = h.process_device_map(d_map, n_dop, n_del, delay, doppler, noise, capi.DET_INTERPOLATE)
        _same((d.delay, d.doppler, d.snr), ref, pos_tol=1e-9)
        assert np.isnan(d.snr).sum() == 1
    h.close()


# ------------------------------------------------------------------------------------------- D: list capacity
def _capacity_map(extra):
    """512 x 1025: spikes on the 512 odd cells of every row (2^18 = the handle's list capacity in all); extra = 1
    moves row 0's spikes to its 513 even cells."""
    m = np.ones((512, 1025), dtype=np.complex64)
    m[:, 1::2] = 100.0
    if extra:
        m[0, :] = 1.0
        m[0, 0::2] = 100.0
    return m


def _det_entry_points(h, m, delay, doppler, cap):
    """(name, rc, n_out, lists, noise power) of b200dd_det_process_device, b200dd_det_process_host (noise power 0) and
    b200dd_det_chain_fetch (the device's Map::set_metrics)."""
    import torch
    lib = h._lib
    n_dop, n_del = m.shape
    delay = np.ascontiguousarray(delay, dtype=np.int32)
    doppler = np.ascontiguousarray(doppler, dtype=np.float64)
    d_map = torch.from_numpy(m).cuda()
    host_map = np.ascontiguousarray(m.astype(np.complex128))
    res = []
    for name in ("process_device", "process_host"):
        out = [np.full(max(1, cap), -7.0) for _ in range(3)]
        n = C.c_uint32(12345)
        if name == "process_device":
            rc = lib.b200dd_det_process_device(h._h, capi.DET_CFAR, capi.ptr(d_map), n_dop, n_del, capi.ptr(delay),
                                               capi.ptr(doppler), 0.0, *(capi.ptr(o) for o in out), cap, C.byref(n), None)
        else:
            rc = lib.b200dd_det_process_host(h._h, capi.DET_CFAR, capi.ptr(host_map), n_dop, n_del, capi.ptr(delay),
                                             capi.ptr(doppler), 0.0, *(capi.ptr(o) for o in out), cap, C.byref(n))
        res.append((name, rc, n.value, out, 0.0))
    rc, k, metrics, out = _chain(h, capi.DET_CFAR, d_map, n_dop, n_del, delay, doppler, cap)
    res.append(("chain_fetch", rc, k, out, metrics[0]))
    return res


def test_detection_list_capacity():
    delay, doppler = _axes(512, 1025)
    h = _det_handle(SPIKES, 512, 1025, 1, 0.5)
    assert h.cap == 1 << 18
    # exactly the capacity: OK and the whole list
    m = _capacity_map(0)
    ref = E.cfar_1d(m, delay, doppler, 0.0, **SPIKES)
    assert ref[0].shape[0] == h.cap
    for name, rc, n, out, noise in _det_entry_points(h, m, delay, doppler, h.cap):
        assert rc == capi.OK and n == h.cap, name
        assert all(np.array_equal(o, r) for o, r in zip(out[:2], ref[:2])), name
        assert np.max(np.abs(out[2] - (ref[2] - noise))) <= 1e-9, name
    # a caller buffer shorter than a valid list: ERR_CAPACITY, n_out = the count, the first `cap` entries filled
    short = 1000
    for name, rc, n, out, _ in _det_entry_points(h, m, delay, doppler, short):
        assert rc == capi.ERR_CAPACITY and n == h.cap, name
        assert all(np.array_equal(o, r[:short]) for o, r in zip(out[:2], ref[:2])), name
    # one detection more than the lists hold: ERR_CAPACITY and n_out = 0
    m = _capacity_map(1)
    assert E.cfar_1d(m, delay, doppler, 0.0, **SPIKES)[0].shape[0] == h.cap + 1
    for name, rc, n, out, _ in _det_entry_points(h, m, delay, doppler, h.cap):
        assert rc == capi.ERR_CAPACITY and n == 0, name
    # the handle still works afterwards
    for name, rc, n, out, _ in _det_entry_points(h, _capacity_map(0), delay, doppler, h.cap):
        assert rc == capi.OK and n == h.cap, name
    h.close()
