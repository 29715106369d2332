"""GPU: the whole-CPI pipeline (C ABI b200dd_pipeline_*) against golden fixtures and the oracle."""
import os

import numpy as np
import pytest

from blah2_b200.process import Pipeline, Ambiguity, WienerHopf
from blah2_b200.scene import make_scene, random_iq, Target
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


@pytest.mark.parametrize("name", ["caf_a", "caf_b", "caf_c"])
def test_cuda_ambiguity_vs_reference_golden(name, relerr):
    d = gold(name)
    geom = tuple(int(v) for v in d["geom"][:6]) + (bool(d["geom"][6]),)
    x, y = random_iq(geom[5], int(d["seed"]))
    m = Ambiguity(*geom).process(x, y)
    e = relerr(m.data, d["map"])
    assert e[0] < 1e-5 and e[1] < 1e-5, e
    assert np.array_equal(m.delay, d["delay"]) and np.array_equal(m.doppler, d["doppler"])


@pytest.mark.parametrize("name", ["wh_a", "wh_b"])
def test_cuda_wienerhopf_vs_reference_golden(name, relerr):
    d = gold(name)
    n, dm, dM, seed = (int(v) for v in d["params"])
    sc = make_scene(n, 2e6, seed=seed, targets=[Target(25, 300.0, -40.0)])
    ok, y = WienerHopf(dm, dM, n).process(sc.x, sc.y)
    assert ok == bool(d["ok"])
    assert relerr(y, d["y"])[0] < 1e-9


def _chain_fixture():
    d = gold("chain_a")
    geom = tuple(int(v) for v in d["geom"][:6]) + (bool(d["geom"][6]),)
    pfa, nGuard, nTrain, minDelay, minDoppler, nCentroid = d["det"]
    det = dict(pfa=float(pfa), nGuard=int(nGuard), nTrain=int(nTrain), minDelay=int(minDelay),
               minDoppler=float(minDoppler), nCentroid=int(nCentroid))
    sc = make_scene(geom[5], geom[4], seed=int(d["seed"]), targets=[Target(17, 300.0, -25.0), Target(41, -200.0, -28.0)])
    return d, geom, det, sc


def test_pipeline_host_vs_reference_golden(relerr):
    d, geom, det, sc = _chain_fixture()
    pipe = Pipeline(*geom[:6], roundHamming=True, clutter=tuple(int(v) for v in d["clutter"]), detection=det)
    out = pipe.process(sc.x, sc.y)
    assert not out["skipped"]
    e = relerr(out["map"], d["map"])
    assert e[0] < 1e-5 and e[1] < 1e-5, e
    assert abs(out["noisePower"] - d["metrics"][0]) < 1e-3 and abs(out["maxPower"] - d["metrics"][1]) < 1e-3
    det_ref = d["interp"]
    got = out["detections"]
    assert got.get_nDetections() == det_ref.shape[1]
    assert np.max(np.abs(got.delay - det_ref[0])) < 1e-3
    assert np.max(np.abs(got.doppler - det_ref[1])) < 1e-3 * abs(d["doppler"][1] - d["doppler"][0]) + 1e-6
    assert np.max(np.abs(got.snr - det_ref[2])) < 1e-3


def test_pipeline_device_path_matches_host_path(relerr):
    import torch
    d, geom, det, sc = _chain_fixture()
    pipe = Pipeline(*geom[:6], roundHamming=True, clutter=tuple(int(v) for v in d["clutter"]), detection=det)
    host = pipe.process(sc.x, sc.y)
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    dmap = torch.empty((pipe.geometry.n_doppler_bins, pipe.geometry.n_delay_bins), dtype=torch.complex64, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):   # back-to-back submissions reuse the handle's buffers
            pipe.submit_device(dx, dy, dmap, s.cuda_stream)
        dev = pipe.fetch(s.cuda_stream)
    assert relerr(dmap.cpu().numpy().astype(np.complex128), host["map"])[0] < 1e-5
    assert dev["detections"].get_nDetections() == host["detections"].get_nDetections()
    assert abs(dev["noisePower"] - host["noisePower"]) < 1e-3


def test_pipeline_without_clutter_or_detection(relerr):
    geom = (-3, 20, -50, 50, 10000, 4000)
    x, y = random_iq(geom[5], 1)
    out = Pipeline(*geom, roundHamming=False).process(x, y)
    ref, _, _ = O.ambiguity_process(x, y, O.ambiguity_geometry(*geom, False))
    assert relerr(out["map"], ref)[0] < 1e-5
    assert out["detections"].get_nDetections() == 0 and not out["skipped"]


def test_pipeline_filter_failure_is_reported():
    n = 8192
    pipe = Pipeline(-3, 20, -50, 50, 10000, n, clutter=(-2, 10), detection=None)
    out = pipe.process(np.zeros(n, complex), np.ones(n, complex))
    assert out["skipped"]


def test_failed_solve_skips_the_cpi_like_the_reference():
    """`if (!filter->process(x, y)) continue;` (blah2.cpp:270-273): with a reference channel whose autocorrelation
    matrix is not positive definite (all zeros) the CPI is skipped -- no detections, no metrics, no map product --
    on the host, int16 and device entry points, although detection is enabled and the surveillance channel is
    full of strong 'targets'."""
    import torch
    n = 8192
    det = dict(pfa=1e-3, nGuard=1, nTrain=4, minDelay=0, minDoppler=0.0, nCentroid=2)
    pipe = Pipeline(-3, 20, -50, 50, 10000, n, clutter=(-2, 10), detection=det)
    rng = np.random.default_rng(5)
    y = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 100.0
    y[::97] += 1e5
    ok_ref, _ = O.wienerhopf_process(np.zeros(n, complex), y, -2, 10)
    assert not ok_ref
    out = pipe.process(np.zeros(n, complex), y)
    assert out["skipped"] and out["detections"].get_nDetections() == 0
    assert out["noisePower"] == 0.0 and out["maxPower"] == 0.0 and out["map"] is None
    dx = torch.zeros(n, dtype=torch.complex64, device="cuda")
    dy = torch.from_numpy(y.astype(np.complex64)).cuda()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        pipe.submit_device(dx, dy, None, s.cuda_stream)
        dev = pipe.fetch(s.cuda_stream)
    assert dev["skipped"] and dev["detections"].get_nDetections() == 0 and dev["noisePower"] == 0.0
    # the next good CPI on the same handle is processed normally
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 100.0
    good = pipe.process(x, 0.5 * x + y * 1e-3)
    assert not good["skipped"] and good["noisePower"] != 0.0


def test_set_metrics_runs_without_detection(relerr):
    """Map::set_metrics follows every Ambiguity::process (blah2.cpp:278-279), detection enabled or not."""
    geom = (-3, 20, -50, 50, 10000, 4000)
    x, y = random_iq(geom[5], 3)
    out = Pipeline(*geom, roundHamming=False).process(x, y)
    noise, mx = O.set_metrics(out["map"])
    assert abs(out["noisePower"] - noise) < 1e-3 and abs(out["maxPower"] - mx) < 1e-3
    assert out["detections"].get_nDetections() == 0


def test_rspduo_int16_ingest_matches_complex128_entry(relerr):
    """N1: the replay layout (int16 I1 Q1 I2 Q2) de-interleaved on the device gives the same CPI result
    as handing over complex128 buffers."""
    d, geom, det, sc = _chain_fixture()
    pipe = Pipeline(*geom[:6], roundHamming=True, clutter=tuple(int(v) for v in d["clutter"]), detection=det)
    host = pipe.process(sc.x, sc.y)
    iq = np.empty((geom[5], 4), dtype="<i2")
    iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = sc.x.real, sc.x.imag, sc.y.real, sc.y.imag
    m = np.empty_like(host["map"])
    pipe.submit_host_rspduo(iq, map_out=m)
    dev = pipe.fetch()
    assert relerr(m, host["map"])[0] < 1e-5
    assert relerr(m, d["map"])[0] < 1e-5
    assert dev["detections"].get_nDetections() == host["detections"].get_nDetections()
    assert np.max(np.abs(dev["detections"].delay - host["detections"].delay)) < 1e-3


def test_graph_replay_of_the_device_chain_is_bit_identical():
    """After b200dd_pipeline_prepare_device a (d_x, d_y, d_map) triple is replayed as one CUDA graph: replayed
    submissions must give the maps, detections and metrics of a pipeline that never prepares (eager) bit for bit --
    also when two prepared triples alternate, when the CONTENT of a buffer changes between replays, and for a CPI
    whose filter fails (status word read after the replay)."""
    import torch
    d, geom, det, sc = _chain_fixture()
    clutter = tuple(int(v) for v in d["clutter"])
    dx = [torch.from_numpy(np.roll(sc.x, 50 * k).astype(np.complex64)).cuda() for k in range(2)]
    dy = [torch.from_numpy(np.roll(sc.y, 50 * k).astype(np.complex64)).cuda() for k in range(2)]

    def run(pipe, k, dmap):
        pipe.submit_device(dx[k], dy[k], dmap)
        r = pipe.fetch()
        return dmap.cpu().numpy().copy(), r

    eager = Pipeline(*geom[:6], roundHamming=True, clutter=clutter, detection=det)
    pipe = Pipeline(*geom[:6], roundHamming=True, clutter=clutter, detection=det)
    shape = (pipe.geometry.n_doppler_bins, pipe.geometry.n_delay_bins)
    em = torch.empty(shape, dtype=torch.complex64, device="cuda")
    gm = [torch.empty(shape, dtype=torch.complex64, device="cuda") for _ in range(2)]
    ref = [run(eager, k, em) for k in range(2)]
    for k in range(2):
        pipe.prepare_device(dx[k], dy[k], gm[k])
    for rep in range(3):          # every submission a replay; the two triples alternate
        for k in range(2):
            m, r = run(pipe, k, gm[k])
            assert np.array_equal(m, ref[k][0]), (rep, k)
            assert r["noisePower"] == ref[k][1]["noisePower"] and r["maxPower"] == ref[k][1]["maxPower"]
            assert np.array_equal(r["detections"].delay, ref[k][1]["detections"].delay)
            assert np.array_equal(r["detections"].snr, ref[k][1]["detections"].snr)
            assert not r["skipped"]
    # new content behind the same pointers: the replay must see it
    dx[0].copy_(dx[1]); dy[0].copy_(dy[1])
    m, r = run(pipe, 0, gm[0])
    assert np.array_equal(m, ref[1][0])
    # a CPI the filter rejects (zero reference channel): reported through the replayed graph as well
    dx[0].zero_()
    m, r = run(pipe, 0, gm[0])
    assert r["skipped"]
    m2, r2 = run(eager, 0, em)
    assert r2["skipped"] and np.array_equal(m, m2)


def test_prepare_device_records_the_graph_up_front():
    """b200dd_pipeline_prepare_device = plan creation: afterwards the FIRST submit of the triple is already a replay and
    gives the result of a pipeline that never prepares (eager) bit for bit, spectrum included.  A triple that was
    never prepared stays eager however often it is submitted."""
    import torch
    d, geom, det, sc = _chain_fixture()
    clutter = tuple(int(v) for v in d["clutter"])
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    outs = {}
    for prepared in (False, True):
        pipe = Pipeline(*geom[:6], roundHamming=True, clutter=clutter, detection=det, spectrum_bandwidth=2000.0)
        dmap = torch.zeros((pipe.geometry.n_doppler_bins, pipe.geometry.n_delay_bins), dtype=torch.complex64, device="cuda")
        scratch = dx.clone()
        if prepared:
            pipe.prepare_device(scratch, dy, dmap)  # runs on whatever the buffers hold now ...
            scratch.copy_(dx)                       # (same values here; the replay reads the buffers when it runs)
            dmap.zero_()
        pipe.submit_device(scratch, dy, dmap)
        r = pipe.fetch()
        outs[prepared] = (dmap.cpu().numpy().copy(), r["noisePower"], r["detections"].delay.copy(), pipe.fetch_spectrum())
        if prepared:                                # an unprepared triple: eager, three times over
            other = torch.zeros_like(dmap)
            for _ in range(3):
                pipe.submit_device(dx, dy, other)
                pipe.fetch()
            assert np.array_equal(other.cpu().numpy(), outs[prepared][0])
    assert np.abs(outs[False][0]).max() > 0
    assert np.array_equal(outs[False][0], outs[True][0]) and outs[False][1] == outs[True][1]
    assert np.array_equal(outs[False][2], outs[True][2]) and np.array_equal(outs[False][3], outs[True][3])
