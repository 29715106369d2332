"""GPU: the FP64 clutter filter on inputs float32 cannot hold, and every entry point at the sample scales of blah2's
other SDR sources.

Part 1.  The complex128 entry points of the clutter filter -- WienerHopf.process, the drop-in WienerHopf class and
the pipeline's host submit, which filters before its complex64 conversion (b200dd_pipeline_submit_host) -- are
FP64 end to end only if they never read their samples through float.  On integer-valued IQ (below 2^24, exact in float32) a narrowing
path gives the same answer, so every input here is unquantised: at least 90 % of its samples change under
astype(np.complex64).  Narrowing x and y moves the filtered output by ~1e-7 relative, far above the filter's 1e-9
bar, but the map by 5e-8 .. 7e-6, under the map's 1e-5 bar: only filter-level checks, a sub-float perturbation and
the pipeline's bit equality with the stage chain can see it.  Every case also asserts that the oracle run on the
complex64-narrowed inputs misses the case's tolerance, so each case is shown to discriminate.

Part 2.  blah2's sources deliver different sample scales: USRP fc32 (floats in +-1, ~2^-15 of the int16 scale) and
HackRF / Kraken int8 (~2^-7).  Scaling by a power of two is exact in floating point (no subnormals or overflow at
these scales) and every stage is linear or ratio-based, so the outputs at x 2^a, y 2^b must be the int16-scale
outputs times an exact power of two, bit for bit.  The detection metrics are logarithmic: noisePower shifts by
(a + b) 10 log10 2 and maxPower does not change, both to rounding.
"""
import importlib.util
import math
import os

import numpy as np
import pytest
import scipy.linalg as sla

from blah2_b200.process import Ambiguity, Pipeline, SpectrumAnalyser, WienerHopf
from blah2_b200.scene import make_scene, Target
from oracle import blah2_oracle as O
from oracle import refpath as R

pytestmark = pytest.mark.gpu

HARNESS = os.path.join(os.path.dirname(R.__file__), "_ref", "libdropin_harness.so")

# the tolerances of test_wh_gpu.test_filter_matches_oracle_fp64_host_path
TOL_AB, TOL_W, TOL_Y, TOL_SOLVE = 1e-12, 1e-9, 1e-9, 1e-10


def _report(case, what, err, bar):
    """One line per tolerance check (pytest -s shows them): the observed error beside its bar."""
    print(f"PRECISION {case} {what}: {err:.3e} (bar {bar:.0e})")


def _c64(a):
    return np.asarray(a).astype(np.complex64)


def _narrowed(a):
    return _c64(a).astype(np.complex128)


def _assert_not_float32(*arrays):
    for a in arrays:
        assert np.mean(_narrowed(a) != a) >= 0.9, "input must not be representable in complex64"


def _gauss(n, seed):
    """Complex Gaussian reference channel and a surveillance channel made of two echoes of it plus noise, each at its
    own random, non-dyadic scale (10^-3 .. 10^3)."""
    rng = np.random.default_rng(seed)
    sx, sy = (rng.uniform(0.55, 1.9) * 10.0 ** int(rng.integers(-3, 4)) for _ in range(2))
    u = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / math.sqrt(2.0)
    v = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / math.sqrt(2.0)
    return sx * u, sy * (0.5 * np.roll(u, 2) + 0.2j * np.roll(u, 17) + 0.05 * v)


def _inputs(kind, n, seed):
    if kind == "scene":
        sc = make_scene(n, 2e6, seed=seed, targets=[Target(25, 300.0, -40.0)], quantise=False)
        x, y = sc.x, sc.y
    else:
        x, y = _gauss(n, seed)
    _assert_not_float32(x, y)
    return x, y


def _filter_case(x, y, dm, dM, case, relerr, wh=None):
    """WienerHopf.process (FP64 host path) against the oracle: a, b, w, y' and the solve of the kernel's own
    Toeplitz system; then the control: the oracle on complex64-narrowed inputs misses the y' bar."""
    wh = wh or WienerHopf(dm, dM, x.shape[0])
    ok, yf = wh.process(x, y)
    ok_ref, w_ref, a_ref, b_ref, xs = O.wienerhopf_weights(x, y, dm, dM)
    assert ok and ok_ref
    w, a, b = wh.debug_weights()
    y_ref = O.wienerhopf_apply(xs, y, w_ref)
    errs = dict(a=(relerr(a, a_ref)[0], TOL_AB), b=(relerr(b, b_ref)[0], TOL_AB), w=(relerr(w, w_ref)[0], TOL_W),
                w_solve=(relerr(w, np.linalg.solve(sla.toeplitz(np.conj(a), a), b))[0], TOL_SOLVE))
    ey = relerr(yf, y_ref)
    errs["y_maxabs"], errs["y_frob"] = (ey[0], TOL_Y), (ey[1], TOL_Y)
    for k, (e, bar) in errs.items():
        _report(case, k, e, bar)
    for k, (e, bar) in errs.items():
        assert e < bar, f"{case} {k}: {e:.3e}"
    ok_n, y_n = O.wienerhopf_process(_narrowed(x), _narrowed(y), dm, dM)
    control = relerr(y_n, y_ref)[0]
    _report(case, "control(narrowed oracle) y_maxabs", control, TOL_Y)
    assert ok_n and control > TOL_Y, f"{case}: complex64-narrowed inputs stay within the bar ({control:.3e})"


# ------------------------------------------------------------------------- part 1: non-representable inputs
# (n, delayMin, delayMax, kind, seed): every solve kernel at both ends of its tap range (1-448 split, 449-480 and
# 481-992 short, 993-1024 and 1025-2048 generic, 2049-4096 long; above 3585 lag blocks and filter partitions),
# delayMin < 0, = 0 and > 0, signals barely longer than the FFT (512, 600: windows wrap and are loaded directly), a
# prime-ish length, and n = 4096 above 3585 taps
FILTER_CASES = [
    (512, 0, 1, "gauss", 1),
    (512, -10, 438, "gauss", 2),
    (600, 7, 40, "gauss", 3),
    (20011, -10, 23, "scene", 4),
    (60000, -10, 438, "scene", 5),
    (60000, 0, 449, "gauss", 6),
    (50021, 5, 485, "scene", 7),
    (50000, -10, 471, "gauss", 8),
    (60000, -10, 982, "scene", 9),
    (60000, 3, 996, "gauss", 10),
    (70000, 0, 1024, "scene", 11),
    (70000, -10, 1015, "gauss", 12),
    (80000, -48, 2000, "scene", 13),
    (80000, 9, 2058, "gauss", 14),
    (60000, -10, 3575, "scene", 15),
    (4096, -10, 3576, "gauss", 16),
    (45000, 9, 4105, "scene", 17),
]


@pytest.mark.parametrize("case", FILTER_CASES, ids=[f"n{c[0]}_taps{c[2] - c[1]}_dmin{c[1]}_{c[3]}" for c in FILTER_CASES])
def test_fp64_filter_on_inputs_float32_cannot_hold(case, relerr):
    n, dm, dM, kind, seed = case
    x, y = _inputs(kind, n, seed)
    _filter_case(x, y, dm, dM, f"taps{dM - dm}_n{n}_dmin{dm}", relerr)


FFT_WINDOWS = {9: (-10, 40), 10: (0, 50), 11: (3, 60), 12: (-5, 70)}


@pytest.mark.parametrize("log2m", [9, 10, 11, 12])
@pytest.mark.parametrize("stage", ["CORR", "APPLY"])
def test_fp64_filter_at_every_fft_length(stage, log2m, relerr, monkeypatch):
    """Every FFT length of the complex128 correlation and filter kernels, forced per stage."""
    monkeypatch.setenv(f"B200DD_WH_{stage}_LOG2M", str(log2m))
    n = 50021
    dm, dM = FFT_WINDOWS[log2m]
    x, y = _inputs("scene" if log2m % 2 else "gauss", n, 100 + log2m)
    wh = WienerHopf(dm, dM, n)
    assert (wh.plan.corr_fft_len if stage == "CORR" else wh.plan.filter_fft_len) == 1 << log2m
    _filter_case(x, y, dm, dM, f"{stage}_M{1 << log2m}", relerr, wh)


def _unit_phase(n, seed):
    return np.exp(2j * np.pi * np.random.default_rng(seed).random(n))


# one tap count per solve kernel (and the partitioned filter at 4096)
PERTURB_TAPS = [(-10, 400), (0, 470), (-10, 690), (3, 1003), (-10, 1490), (-50, 2950), (9, 4105)]


@pytest.mark.parametrize("window", PERTURB_TAPS, ids=[f"taps{b - a}" for a, b in PERTURB_TAPS])
def test_sub_float_perturbations_reach_the_output(window, relerr):
    """The filter is linear in y for fixed x: WH(x, y + d) - WH(x, y) = WH(x, d) for a d of 2^-30 max|y|, below
    float32's resolution of y (most samples of y + d round back to y).  A perturbation of x of the same relative size
    must move the output as it moves the oracle's.  A path that narrows its inputs loses both."""
    dm, dM = window
    n = 60000
    x, y = _inputs("gauss" if dm else "scene", n, dM)
    d = (2.0 ** -30 * np.max(np.abs(y))) * _unit_phase(n, 1)
    e = (2.0 ** -30 * np.max(np.abs(x))) * _unit_phase(n, 2)
    assert np.mean(_c64(y + d) == _c64(y)) > 0.5 and np.mean(_c64(x + e) == _c64(x)) > 0.5
    wh = WienerHopf(dm, dM, n)
    outs = {}
    for k, (xi, yi) in dict(base=(x, y), dy=(x, y + d), d=(x, d), dx=(x + e, y)).items():
        ok, outs[k] = wh.process(xi, yi)
        assert ok, k
    case = f"perturb_taps{dM - dm}"
    lin = np.max(np.abs((outs["dy"] - outs["base"]) - outs["d"])) / np.max(np.abs(outs["d"]))
    ref_dx = O.wienerhopf_process(x + e, y, dm, dM)[1] - O.wienerhopf_process(x, y, dm, dM)[1]
    ex = relerr(outs["dx"] - outs["base"], ref_dx)[0]
    _report(case, "WH(x,y+d)-WH(x,y) vs WH(x,d)", lin, 1e-5)
    _report(case, "WH(x+e,y)-WH(x,y) vs oracle", ex, 1e-4)
    assert lin < 1e-5 and ex < 1e-4, (lin, ex)
    # controls: the oracle on narrowed inputs misses both bars
    on = {k: O.wienerhopf_process(_narrowed(xi), _narrowed(yi), dm, dM)[1]
          for k, (xi, yi) in dict(base=(x, y), dy=(x, y + d), d=(x, d), dx=(x + e, y)).items()}
    c_lin = np.max(np.abs((on["dy"] - on["base"]) - on["d"])) / np.max(np.abs(on["d"]))
    c_ex = relerr(on["dx"] - on["base"], ref_dx)[0]
    _report(case, "control(narrowed oracle) y-perturbation", c_lin, 1e-5)
    _report(case, "control(narrowed oracle) x-perturbation", c_ex, 1e-4)
    assert c_lin > 1e-5 and c_ex > 1e-4, (c_lin, c_ex)


@pytest.fixture(scope="module")
def D():
    """The refpath binding pointed at the drop-in harness (test_dropin_gpu.py)."""
    if not os.path.exists(HARNESS):
        pytest.fail(f"{HARNESS} missing: build() makes it where the blah2 sources exist (/root/reference or BLAH2_SRC)")
    spec = importlib.util.spec_from_file_location("dropin_binding_precision", R.__file__)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.LIB_PATH = HARNESS
    return mod


DROPIN_CASES = [(60011, -10, 60, "scene", 31), (100003, 3, 500, "gauss", 32), (300000, -50, 2000, "gauss", 33)]


@pytest.mark.parametrize("case", DROPIN_CASES, ids=[f"taps{c[2] - c[1]}_dmin{c[1]}_{c[3]}" for c in DROPIN_CASES])
def test_dropin_wienerhopf_on_inputs_float32_cannot_hold(D, case, relerr):
    n, dm, dM, kind, seed = case
    x, y = _inputs(kind, n, seed)
    ok, yf = D.wienerhopf_process(x, y, dm, dM)
    ref = R.wienerhopf_process if R.available() else O.wienerhopf_process
    ok_ref, y_ref = ref(x, y, dm, dM)
    assert ok and ok_ref
    e = relerr(yf, y_ref)
    name = f"dropin_taps{dM - dm}_dmin{dm}"
    _report(name, "y_maxabs", e[0], TOL_Y)
    _report(name, "y_frob", e[1], TOL_Y)
    assert e[0] < TOL_Y and e[1] < TOL_Y, e
    control = relerr(ref(_narrowed(x), _narrowed(y), dm, dM)[1], y_ref)[0]
    _report(name, "control(narrowed reference) y_maxabs", control, TOL_Y)
    assert control > TOL_Y


CONFIG2_DET = dict(pfa=1e-5, nGuard=2, nTrain=6, minDelay=5, minDoppler=15.0, nCentroid=6)


def _device_chain(geom, det, x32, y32):
    """Ambiguity.process_device and a clutter-free pipeline's submit_device on the same complex64 channels: (map,
    pipeline map, pipeline result)."""
    import torch
    dx, dy = torch.from_numpy(x32).cuda(), torch.from_numpy(y32).cuda()
    amb = Ambiguity(*geom)
    g = amb.geometry
    shape = (g.n_doppler_bins, g.n_delay_bins)
    m = torch.empty(shape, dtype=torch.complex64, device="cuda")
    torch.cuda.synchronize()
    amb.process_device(dx, dy, m)
    torch.cuda.synchronize()
    pipe = Pipeline(*geom[:6], roundHamming=geom[6], detection=det)
    pm = torch.empty(shape, dtype=torch.complex64, device="cuda")
    pipe.submit_device(dx, dy, pm)
    r = pipe.fetch()
    return m.cpu().numpy(), pm.cpu().numpy(), r


@pytest.mark.parametrize("clutter", [(-10, 400), (-50, 2000)])
def test_pipeline_host_submit_equals_the_fp64_stage_chain(clutter):
    """Pipeline.submit_host on complex128 samples float32 cannot hold = WienerHopf.process (FP64), the filtered y
    rounded to complex64, then the CAF, set_metrics and detection on the device -- map, metrics and detections bit for
    bit.  The map's 1e-5 bar cannot see a narrowing of the inputs before the filter; this equality can."""
    geom = (0, 299, -128, 128, 2000000, 400000, True)
    n = geom[5]
    sc = make_scene(n, geom[4], seed=2026, quantise=False)
    x, y = sc.x, sc.y
    _assert_not_float32(x, y)
    pipe = Pipeline(*geom[:6], roundHamming=True, clutter=clutter, detection=CONFIG2_DET)
    got = np.empty((pipe.geometry.n_doppler_bins, pipe.geometry.n_delay_bins), dtype=np.complex128)
    pipe.submit_host(x, y, map_out=got)
    r = pipe.fetch()
    assert not r["skipped"]

    def stage_chain(xi, yi):
        ok, yf = WienerHopf(*clutter, n).process(xi, yi)
        assert ok
        return _device_chain(geom, CONFIG2_DET, _c64(xi), _c64(yf))

    m, pm, sr = stage_chain(x, y)
    assert np.array_equal(got, m.astype(np.complex128))
    assert np.array_equal(pm, m)
    assert r["noisePower"] == sr["noisePower"] and r["maxPower"] == sr["maxPower"]
    d, sd = r["detections"], sr["detections"]
    assert d.get_nDetections() == sd.get_nDetections() >= 2
    for f in ("delay", "doppler", "snr"):
        assert np.array_equal(getattr(d, f), getattr(sd, f)), f
    # control: the same chain on complex64-narrowed inputs gives another map
    mn = stage_chain(_narrowed(x), _narrowed(y))[0]
    diff = np.max(np.abs(mn.astype(np.complex128) - m)) / np.max(np.abs(m))
    _report(f"pipeline_host_clutter{clutter[1] - clutter[0]}", "control(narrowed chain) map", diff, 0.0)
    assert diff > 0.0


# --------------------------------------------------------------------- part 2: fc32 and int8 sample scales
# (a, b): x 2^a, y 2^b.  (-15, -15) is USRP fc32 scale, (-7, -7) int8 scale.
SCALES = [(-15, -15), (-15, -8), (-7, -7), (10, 4)]
SCALE_IDS = [f"x2^{a}_y2^{b}" for a, b in SCALES]
GEOM_SYM = (0, 299, -128, 128, 2000000, 400000, True)     # blah2's config 2 at a fifth of its CPI
GEOM_OFF = (0, 299, -60, 196, 2000000, 400000, True)      # off-centre Doppler window (pre-rotated reference)
CLUTTER = (-10, 400)
BANDWIDTH = 2000.0
LOG2_DB = 10.0 * math.log10(2.0)


@pytest.fixture(scope="module")
def int16_scene():
    sc = make_scene(GEOM_SYM[5], GEOM_SYM[4], seed=20261017,
                    targets=[Target(37, 55.0, -45.0), Target(92, -103.0, -50.0), Target(151, 78.0, -55.0),
                             Target(230, -41.0, -50.0), Target(60, 40.0, -35.0)])
    assert np.array_equal(_narrowed(sc.x), sc.x) and np.array_equal(_narrowed(sc.y), sc.y)
    return sc


def _scaled(v, k):
    return v * (2.0 ** k)


def _wh_outputs(x, y):
    """(host complex128 output, device complex64 output) of the clutter filter."""
    import torch
    wh = WienerHopf(*CLUTTER, x.shape[0])
    ok, host = wh.process(x, y)
    assert ok
    dx, dy = torch.from_numpy(_c64(x)).cuda(), torch.from_numpy(_c64(y)).cuda()
    out = torch.empty_like(dy)
    torch.cuda.synchronize()
    wh.process_device(dx, dy, out)
    torch.cuda.synchronize()
    assert wh.last_status()
    return host, out.cpu().numpy()


@pytest.fixture(scope="module")
def filtered(int16_scene):
    return _wh_outputs(int16_scene.x, int16_scene.y)


@pytest.mark.parametrize("a,b", SCALES, ids=SCALE_IDS)
def test_clutter_filter_is_scale_equivariant(a, b, int16_scene, filtered):
    host, dev = _wh_outputs(_scaled(int16_scene.x, a), _scaled(int16_scene.y, b))
    assert np.array_equal(host, _scaled(filtered[0], b))
    assert np.array_equal(dev, _c64(_scaled(filtered[1].astype(np.complex128), b)))


def _caf_maps(geom, x, y):
    """(host map, device map) of Ambiguity on complex64-exact channels."""
    import torch
    amb = Ambiguity(*geom)
    host = amb.process(x, y).data
    g = amb.geometry
    dm = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    dx, dy = torch.from_numpy(_c64(x)).cuda(), torch.from_numpy(_c64(y)).cuda()
    torch.cuda.synchronize()
    amb.process_device(dx, dy, dm)
    torch.cuda.synchronize()
    return host, dm.cpu().numpy().astype(np.complex128)


@pytest.mark.parametrize("geom", [GEOM_SYM, GEOM_OFF], ids=["symmetric", "off_centre"])
@pytest.mark.parametrize("a,b", SCALES, ids=SCALE_IDS)
def test_caf_is_scale_equivariant(a, b, geom, int16_scene, filtered):
    y = filtered[1].astype(np.complex128)   # the filtered surveillance channel, complex64-exact
    base = _caf_maps(geom, int16_scene.x, y)
    got = _caf_maps(geom, _scaled(int16_scene.x, a), _scaled(y, b))
    for g, r, path in zip(got, base, ("host", "device")):
        assert np.all(np.isfinite(r)) and np.max(np.abs(r)) > 0
        assert np.array_equal(g, _scaled(r, a + b)), path


@pytest.mark.parametrize("a", sorted({a for a, _ in SCALES}))
def test_spectrum_is_scale_equivariant(a, int16_scene):
    import torch
    x = int16_scene.x
    sa = SpectrumAnalyser(x.shape[0], BANDWIDTH)

    def run(v):
        host = sa.process(v)[0]
        out = []
        for t in (torch.from_numpy(_c64(v)).cuda(), torch.from_numpy(v.copy()).cuda()):   # float2 and double2 input
            torch.cuda.synchronize()
            sa.process_device(t)
            out.append(sa.fetch())
        return [host] + out

    for g, r in zip(run(_scaled(x, a)), run(x)):
        assert np.array_equal(g, _scaled(r, a))


def _pipeline_runs(x, y):
    """The CPI through submit_host, submit_device (eager) and submit_device replayed as a CUDA graph: per entry point
    (map as complex128, fetch result, spectrum)."""
    import torch

    def make():
        return Pipeline(*GEOM_SYM[:6], roundHamming=True, clutter=CLUTTER, detection=CONFIG2_DET,
                        spectrum_bandwidth=BANDWIDTH)

    runs = {}
    p = make()
    m = np.empty((p.geometry.n_doppler_bins, p.geometry.n_delay_bins), dtype=np.complex128)
    p.submit_host(np.ascontiguousarray(x), np.ascontiguousarray(y), map_out=m)
    r = p.fetch()
    runs["submit_host"] = (m, r, p.fetch_spectrum())
    dx, dy = torch.from_numpy(_c64(x)).cuda(), torch.from_numpy(_c64(y)).cuda()
    for name in ("submit_device", "graph_replay"):
        p = make()
        dm = torch.empty(m.shape, dtype=torch.complex64, device="cuda")
        if name == "graph_replay":
            p.prepare_device(dx, dy, dm)
            dm.zero_()
        p.submit_device(dx, dy, dm)
        r = p.fetch()
        runs[name] = (dm.cpu().numpy().astype(np.complex128), r, p.fetch_spectrum())
    for name, (_, r, _) in runs.items():
        assert not r["skipped"] and r["detections"].get_nDetections() >= 2, name
    return runs


@pytest.fixture(scope="module")
def pipeline_base(int16_scene):
    return _pipeline_runs(int16_scene.x, int16_scene.y)


@pytest.mark.parametrize("a,b", SCALES, ids=SCALE_IDS)
def test_pipeline_is_scale_equivariant(a, b, int16_scene, pipeline_base):
    """Map 2^(a+b), spectrum 2^a bit for bit; the same detections (the CFAR compares |z z| sums, which scale exactly);
    noisePower shifted by (a + b) 10 log10 2 (Map::set_metrics averages 10 log10|z|); maxPower unchanged while the
    largest cell stays above 0 dB, where the reference's running maximum starts (Map.cpp:193)."""
    runs = _pipeline_runs(_scaled(int16_scene.x, a), _scaled(int16_scene.y, b))
    for name, (m, r, spec) in runs.items():
        m0, r0, spec0 = pipeline_base[name]
        assert np.array_equal(m, _scaled(m0, a + b)), name
        assert np.array_equal(spec, _scaled(spec0, a)), name
        assert r["noisePower"] + r["maxPower"] > 0.0, name   # the largest cell is above 0 dB at this scale
        d, d0 = r["detections"], r0["detections"]
        assert d.get_nDetections() == d0.get_nDetections(), name
        errs = dict(delay=np.max(np.abs(d.delay - d0.delay)), doppler=np.max(np.abs(d.doppler - d0.doppler)),
                    snr=np.max(np.abs(d.snr - d0.snr)),
                    noisePower=abs(r["noisePower"] - r0["noisePower"] - (a + b) * LOG2_DB),
                    maxPower=abs(r["maxPower"] - r0["maxPower"]))
        for k, e in errs.items():
            _report(f"pipeline_{name}_x2^{a}_y2^{b}", k, e, 1e-9)
        assert all(e <= 1e-9 for e in errs.values()), (name, errs)


def test_fc32_scale_scene_against_the_oracle_chain(int16_scene, relerr):
    """The int16 scene at USRP fc32 scale (x 2^-15) through the whole pipeline against the numpy chain."""
    x, y = _scaled(int16_scene.x, -15), _scaled(int16_scene.y, -15)
    out = Pipeline(*GEOM_SYM[:6], roundHamming=True, clutter=CLUTTER, detection=CONFIG2_DET).process(x, y)
    ref = O.chain(x, y, O.ambiguity_geometry(*GEOM_SYM), clutter=CLUTTER, det=CONFIG2_DET)
    assert not out["skipped"] and not ref["skipped"]
    e = relerr(out["map"], ref["map"])
    _report("fc32_scene", "map_maxabs", e[0], 1e-5)
    _report("fc32_scene", "map_frob", e[1], 1e-5)
    assert e[0] < 1e-5 and e[1] < 1e-5, e
    assert abs(out["noisePower"] - ref["noisePower"]) < 1e-3 and abs(out["maxPower"] - ref["maxPower"]) < 1e-3
    d, rd = out["detections"], ref["detections"]
    assert d.get_nDetections() == len(rd[0]) >= 2
    res = GEOM_SYM[4] / GEOM_SYM[5]
    assert np.max(np.abs(d.delay - rd[0])) < 1e-3
    assert np.max(np.abs(d.doppler - rd[1])) < 1e-3 * res
    assert np.max(np.abs(d.snr - rd[2])) < 1e-3
