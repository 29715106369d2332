"""GPU: the clutter filter above 2048 taps (2049-4096): the long solve kernel, the lag-block correlations and the
partitioned overlap-save filter.

* Against tests/golden/wh_long_*.npz, written by the reference's unmodified WienerHopf::process
  (oracle/gen_golden_wh_long.py): a and b to 1e-12, w and the FP64 y' to 1e-9, the reference's verdict (and untouched
  y) where its chol() fails; the float2 y' to 1e-6 of the FP64 filter of the same complex64 inputs.
* Against the numpy restatement (oracle/blah2_oracle.py) run live at 2050 and 3586 taps.
* The new kernels on 16- and 8-byte misaligned, NaN-guarded buffers; chunk mode emulating three ranks; a pipeline at
  2050 clutter taps against the stage-by-stage chain, eager and graph-replayed; the drop-in class at 2050 taps.
"""
import glob
import os

import numpy as np
import pytest

from blah2_b200.process import Ambiguity, Pipeline, WienerHopf
from blah2_b200.scene import make_scene, Target
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = sorted(glob.glob(os.path.join(GOLDEN, "wh_long_*.npz")))


def _fixture_inputs(d):
    n, seed = int(d["N"]), int(d["seed"])
    if seed < 0:
        return np.zeros(n, dtype=np.complex128), make_scene(n, 2000000, seed=4100).y
    sc = make_scene(n, 2000000, seed=seed)
    return sc.x, sc.y


def _projection(n, seed=7):
    rng = np.random.default_rng(seed)
    return np.exp(2j * np.pi * rng.random(n))


def _check_y(y, d, tol, relerr):
    step = int(d["step"])
    assert relerr(y[::step], d["sub"])[0] < tol
    assert abs(np.linalg.norm(y) - float(d["norm"])) < tol * float(d["norm"])
    proj = np.sum(y * _projection(y.shape[0]))
    assert abs(proj - complex(d["proj"])) < tol * float(d["norm"]) * np.sqrt(y.shape[0])


def _sync():
    import torch
    torch.cuda.synchronize()


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[8:-4] for p in FIXTURES])
def test_filter_matches_the_reference_fixtures(path, relerr):
    import torch
    d = np.load(path)
    dm, dM, n = int(d["delayMin"]), int(d["delayMax"]), int(d["N"])
    x, y = _fixture_inputs(d)
    wh = WienerHopf(dm, dM, n)
    nb = dM - dm
    p = wh.plan
    assert wh.nBins == nb and p.solve_rows_per_thread == 4 and p.solve_threads == (nb + 127) // 128 * 32
    assert (p.corr_lag_blocks, p.filter_partitions) == ((2, 2) if nb > 3585 else (1, 1))
    # FP64 host path (y and y' in one buffer)
    ok, yf = wh.process(x, y)
    assert ok == bool(d["ok"])
    w, a, b = wh.debug_weights()
    for got, ref in ((a, d["a"]), (b, d["b"])):   # (an all-zero reference channel has a = 0 exactly)
        assert relerr(got, ref)[0] < 1e-12 if np.any(ref) else not np.any(got)
    if not ok:
        assert np.array_equal(yf, y)
        return
    assert relerr(w, d["w"])[0] < 1e-9
    _check_y(yf, d, 1e-9, relerr)
    # float2 device path: its inputs are the complex64 roundings of x and y (the scene's y is not float32-exact, and
    # 30-60 dB of cancellation amplify that rounding), so its yardstick is the FP64 filter of the same rounded inputs,
    # which the lines above pin to the reference
    x32, y32 = x.astype(np.complex64), y.astype(np.complex64)
    ok64, y64 = wh.process(x32.astype(np.complex128), y32.astype(np.complex128))
    dx, dy = torch.from_numpy(x32).cuda(), torch.from_numpy(y32).cuda()
    out = torch.empty_like(dy)
    _sync()
    wh.process_device(dx, dy, out)
    _sync()
    assert ok64 and wh.last_status()
    e = relerr(out.cpu().numpy().astype(np.complex128), y64)
    assert e[0] < 1e-6 and e[1] < 1e-6, e


def test_failed_solve_leaves_the_device_output_untouched():
    import torch
    d = np.load(os.path.join(GOLDEN, "wh_long_fail4096.npz"))
    dm, dM, n = int(d["delayMin"]), int(d["delayMax"]), int(d["N"])
    x, y = _fixture_inputs(d)
    wh = WienerHopf(dm, dM, n)
    dy = torch.from_numpy(y.astype(np.complex64)).cuda()
    out = torch.full_like(dy, complex(7, 7))
    _sync()
    wh.process_device(torch.zeros_like(dy), dy, out)
    _sync()
    assert not wh.last_status()
    assert np.array_equal(out.cpu().numpy(), y.astype(np.complex64))   # pass-through of y, as the reference leaves it


@pytest.mark.parametrize("case", [(300000, -50, 2000, 11), (200000, 3, 3589, 12)])
def test_filter_matches_the_numpy_restatement(case, relerr):
    n, dm, dM, seed = case
    sc = make_scene(n, 2e6, seed=seed, targets=[Target(25, 300.0, -40.0)])
    wh = WienerHopf(dm, dM, n)
    ok, y = wh.process(sc.x, sc.y)
    ok_ref, w_ref, a_ref, b_ref, xs = O.wienerhopf_weights(sc.x, sc.y, dm, dM)
    assert ok and ok_ref
    w, a, b = wh.debug_weights()
    assert relerr(a, a_ref)[0] < 1e-12 and relerr(b, b_ref)[0] < 1e-12
    assert relerr(w, w_ref)[0] < 1e-9
    e = relerr(y, O.wienerhopf_apply(xs, sc.y, w_ref))
    assert e[0] < 1e-9 and e[1] < 1e-9, e


# one case per new kernel combination: long solve with the one-block plans (2050, 3000), lag blocks and partitions
# (3586, 4096); delayMin < 0, = 0 and > 0 (> 0: windows loaded through the reference's index map, not staged)
MISALIGNED = [(60000, -50, 2000), (50000, 0, 3000), (40000, -6, 3580), (50000, 0, 4096), (45000, 9, 4105)]


@pytest.mark.parametrize("case", MISALIGNED, ids=[f"{c[2] - c[1]}taps_dmin{c[1]}" for c in MISALIGNED])
def test_new_kernels_on_misaligned_guarded_buffers(case, relerr):
    from test_kernel_edges_gpu import _c64, _wh_check
    n, dm, dM = case
    sc = make_scene(n, 2e6, seed=n + dM, targets=[Target(25, 300.0, -40.0)])
    wh = WienerHopf(dm, dM, n)
    _wh_check(wh, _c64(sc.x), _c64(sc.y), dm, dM, relerr)


@pytest.mark.parametrize("case", [(400000, -50, 2000, 3, 21), (500000, -100, 3996, 3, 22)])
def test_chunked_filter_emulating_three_ranks(case, relerr):
    import torch
    from blah2_b200.process import WienerHopfChunk
    from blah2_b200.shard import block_range
    n, dm, dM, world, seed = case
    sc = make_scene(n, 2e6, seed=seed, targets=[Target(25, 300.0, -40.0)])
    xg, yg = sc.x.astype(np.complex64), sc.y.astype(np.complex64)
    wh = WienerHopf(dm, dM, n)
    whole = torch.empty(n, dtype=torch.complex64, device="cuda")
    _sync()
    wh.process_device(torch.from_numpy(xg).cuda(), torch.from_numpy(yg).cuda(), whole)
    _sync()
    w_ref, a_ref, b_ref = wh.debug_weights()
    chunks, abs_ = [], []
    for r in range(world):
        c0, nc = block_range(n, r, world)
        ch = WienerHopfChunk(dm, dM, n, c0, nc)
        xl, xr, yr = ch.halos()
        assert (xl, xr, yr) == (max(dM - dm - 1 + dm, 0), dM - dm - 1 - dm, dM - dm - 1)
        x_loc = torch.from_numpy(xg[np.arange(c0 - xl, c0 + nc + xr) % n]).cuda()
        y_loc = torch.from_numpy(yg[np.arange(c0, c0 + nc + yr) % n]).cuda()
        ab = torch.zeros(2 * ch.nBins, dtype=torch.complex128, device="cuda")
        ch.corr_device(x_loc, y_loc, ab)
        chunks.append((ch, x_loc, y_loc, nc))
        abs_.append(ab)
    _sync()
    ab_sum = torch.stack(abs_).sum(0)
    nb = dM - dm
    assert relerr(ab_sum[:nb].cpu().numpy(), a_ref)[0] < 1e-12 and relerr(ab_sum[nb:].cpu().numpy(), b_ref)[0] < 1e-12
    outs = []
    for ch, x_loc, y_loc, nc in chunks:
        o = torch.empty(nc, dtype=torch.complex64, device="cuda")
        ch.filter_device(ab_sum, x_loc, y_loc, o)
        outs.append(o)
    _sync()
    assert all(c[0].last_status() for c in chunks)
    got = torch.cat(outs).cpu().numpy()
    assert relerr(got, whole.cpu().numpy())[0] < 1e-6
    ok, y_ref = O.wienerhopf_process(xg.astype(np.complex128), yg.astype(np.complex128), dm, dM)
    assert ok and relerr(got, y_ref)[0] < 1e-6


def test_pipeline_at_2050_clutter_taps_equals_the_stage_chain(relerr):
    """Pipeline(clutter=(-50, 2000)) -- blah2's default window at 10 MS/s -- against WienerHopf -> Ambiguity on the
    device (bit for bit), against the numpy chain (map and detections), eager and graph-replayed (bit for bit)."""
    import torch
    geom = (-10, 120, -300, 300, 2000000, 400000, True)
    clutter = (-50, 2000)
    det = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
    sc = make_scene(geom[5], geom[4], seed=41, targets=[Target(37, 110.0, -40.0), Target(92, -205.0, -45.0)])
    x, y = sc.x.astype(np.complex64), sc.y.astype(np.complex64)
    dx, dy = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    # stage by stage
    wh = WienerHopf(*clutter, geom[5])
    amb = Ambiguity(*geom)
    g = amb.geometry
    shape = (g.n_doppler_bins, g.n_delay_bins)
    yf = torch.empty_like(dy)
    stage_map = torch.empty(shape, dtype=torch.complex64, device="cuda")
    s = torch.cuda.Stream()   # one stream: the map stage reads what the filter wrote
    _sync()
    wh.process_device(dx, dy, yf, s.cuda_stream)
    amb.process_device(dx, yf, stage_map, s.cuda_stream)
    s.synchronize()
    stage_map = stage_map.cpu().numpy()
    # eager pipeline, then a graph-replayed one
    eager = Pipeline(*geom[:6], roundHamming=True, clutter=clutter, detection=det)
    em = torch.empty(shape, dtype=torch.complex64, device="cuda")
    eager.submit_device(dx, dy, em)
    er = eager.fetch()
    assert not er["skipped"]
    assert np.array_equal(em.cpu().numpy(), stage_map)
    pipe = Pipeline(*geom[:6], roundHamming=True, clutter=clutter, detection=det)
    gm = torch.empty(shape, dtype=torch.complex64, device="cuda")
    pipe.prepare_device(dx, dy, gm)
    for _ in range(2):
        pipe.submit_device(dx, dy, gm)
        r = pipe.fetch()
        assert np.array_equal(gm.cpu().numpy(), stage_map)
        assert r["noisePower"] == er["noisePower"] and r["maxPower"] == er["maxPower"]
        assert np.array_equal(r["detections"].delay, er["detections"].delay)
        assert np.array_equal(r["detections"].doppler, er["detections"].doppler)
        assert np.array_equal(r["detections"].snr, er["detections"].snr)
    # the numpy chain on the same float32 inputs
    ref = O.chain(x.astype(np.complex128), y.astype(np.complex128), O.ambiguity_geometry(*geom), clutter=clutter, det=det)
    assert not ref["skipped"]
    assert relerr(stage_map.astype(np.complex128), ref["map"])[0] < 1e-5
    d, rd = er["detections"], ref["detections"]
    assert d.get_nDetections() == len(rd[0]) and d.get_nDetections() >= 2
    assert np.max(np.abs(d.delay - rd[0])) < 1e-3 and np.max(np.abs(d.snr - rd[2])) < 1e-3


def test_dropin_wienerhopf_at_2050_taps(relerr):
    """The C++ drop-in WienerHopf class (same source-level API as the reference's) at blah2's default 10 MS/s window,
    against the reference class where it is built, else the numpy restatement."""
    import importlib.util
    from oracle import refpath as R
    harness = os.path.join(os.path.dirname(R.__file__), "_ref", "libdropin_harness.so")
    if not os.path.exists(harness):
        pytest.fail(f"{harness} missing: build() makes it where the blah2 sources exist (/root/reference or BLAH2_SRC)")
    spec = importlib.util.spec_from_file_location("dropin_binding_long", R.__file__)
    D = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(D)
    D.LIB_PATH = harness
    sc = make_scene(300000, 10e6, seed=43)
    ok, y = D.wienerhopf_process(sc.x, sc.y, -50, 2000)
    ok_ref, y_ref = (R.wienerhopf_process if R.available() else O.wienerhopf_process)(sc.x, sc.y, -50, 2000)
    assert ok and ok_ref
    e = relerr(y, y_ref)
    assert e[0] < 1e-9 and e[1] < 1e-9, e
