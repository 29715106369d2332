"""GPU: the drop-in SpectrumAnalyser, CfarDetector1D, Centroid, Interpolate, Ambiguity and WienerHopf against blah2's
own classes, through one class harness (oracle/dropinclass/class_capi.cpp) built with each.  Every object is created
once and called over a sequence of inputs, as blah2.cpp calls its objects once per CPI, so the state a class keeps
between calls is what is tested: the detection handles the drop-ins reuse while a map is no larger than the last
rebuild, Centroid's fixed handle, the samples Ambiguity leaves queued and rotates, and the surveillance FIFO
WienerHopf replaces.  The whole blah2.cpp loop body runs over 25 consecutive CPIs through oracle/refpath.

Bars, from where each value is exact:
  bit for bit   CFAR's delay and Doppler lists (|z z| against the training mean in FP64), Centroid's lists, every
                sample Ambiguity leaves in either FIFO without a clutter filter and in x with one, FIFO lengths,
                get_n_samples(), the frequency vector, and y after a failed solve;
  dB values     CFAR's SNRs and Interpolate's lists go through CUDA's log10 where the reference calls glibc's.  They
                must equal det_cases' restatement fed the device's own per-cell dB values bit for bit, and lie
                within db_bound (derived below) of the reference;
  envelopes     the spectrum against numpy's FP64 FFT within tests/test_spectrum_envelope_gpu.py's error model, the
                map 1e-5 and the filtered channel 1e-9 of the reference, as tests/test_dropin_gpu.py.
"""
import importlib.util
import math
import os
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import det_cases as D  # noqa: E402
import dropin_class_cases as K  # noqa: E402
import spectrum_cases as S  # noqa: E402

from oracle import blah2_oracle as O  # noqa: E402
from oracle import dropin_class as DC  # noqa: E402
from oracle import refpath as R  # noqa: E402

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not (DC.available("ref") and DC.available("dropin")),
                                 reason="class harnesses not built (build() with the blah2 sources)")]
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module", autouse=True)
def _report_runtime():
    t0 = time.perf_counter()
    yield
    print(f"\ntest_dropin_classes_gpu: {time.perf_counter() - t0:.1f} s")


def _both(cls, *args):
    return cls("ref", *args), cls("dropin", *args)


# ---------------------------------------------------------------------------------------------- dB values
def dev_db(m, delay, doppler, noise):
    """cell_db of every cell as the device computes it (10 log10 hypot(re, im) - noisePower)."""
    from blah2_b200.process import MapJson

    mj = MapJson(delay, doppler, 2000000)
    try:
        return mj.cell_values(torch.from_numpy(np.ascontiguousarray(m, np.complex128)).cuda(), noise)
    finally:
        mj.close()


def db_bound(db_cpu, noise):
    """How far a cell's dB value on the device can lie from the reference's, from the libraries' documented errors.

    |z| is hypot on both sides: CUDA's hypot is within 2 ulp (CUDA C Programming Guide, double-precision functions),
    glibc's within 1 ulp (glibc manual, "Known Maximum Errors in Math Functions", x86_64), so the two magnitudes differ
    by a factor within 1 +- 3 * 2^-52, and their log10 by at most 3 * 2^-52 / ln 10 (plus its square, far below).
    log10 is within 1 ulp on CUDA and 2 ulp in glibc: 3 ulp(L) more, counted as 6 ulp(|L|) in case L and the true
    value lie in different binades.  10 L is rounded on each side (1 ulp of 10 |L| between them, 2 across a binade),
    and so is the subtraction of noisePower (2 ulp of the result):

        |db_dev - db_ref| <= 10 (6 ulp(|L|) + 3.01 * 2^-52 / ln 10) + 2 ulp(10 |L|) + 2 ulp(|db|)

    with L = (db_ref + noisePower) / 10.  No constant here is fitted to a measurement."""
    L = np.abs((np.asarray(db_cpu, np.float64) + noise) / 10.0)
    ulp = np.vectorize(math.ulp, otypes=[np.float64])
    return (10.0 * (6.0 * ulp(L) + 3.01 * 2.0 ** -52 / math.log(10.0)) + 2.0 * ulp(10.0 * L)
            + 2.0 * ulp(np.abs(db_cpu)))


def assert_db_close(db_dev, db_cpu, noise):
    fin = np.isfinite(db_cpu)
    assert np.array_equal(np.isfinite(db_dev), fin)
    err = np.abs(db_dev[fin] - db_cpu[fin])
    assert np.all(err <= db_bound(db_cpu[fin], noise)), float(np.max(err / db_bound(db_cpu[fin], noise)))


def same(a, b):
    return D.same(a, b)


# ---------------------------------------------------------------------------------------------- SpectrumAnalyser
@pytest.mark.parametrize("r", S.ROWS, ids=S.row_id)
def test_spectrum_analyser_over_consecutive_fifos(r):
    from blah2_b200.process import SpectrumAnalyser
    from test_spectrum_envelope_gpu import error_bar, make_input

    ref, dro = _both(DC.SpectrumAnalyserClass, r["n"], r["bw"])
    sa = SpectrumAnalyser(r["n"], r["bw"])
    geom = sa.geometry
    sa.close()
    try:
        for k in range(2):  # one object, two FIFOs of different contents
            x, _ = make_input(r, seed=r["n_spectrum"] * 31 + r["dec"] + 1000 * k)
            want, freq = O.spectrum_process(x.astype(np.complex128), r["n"], r["bw"])
            s_ref, f_ref, left_ref = ref.process(x)
            s, f, left = dro.process(x)
            assert left == left_ref == r["n"]                       # process reads the FIFO, never pops it
            assert f.size == f_ref.size == freq.size == 0           # the reference's uint32_t loop never runs
            assert s.shape == s_ref.shape == want.shape
            bar = error_bar(r, geom, x)
            err = np.abs(s - want)
            assert np.all(err <= bar), (k, float(np.max(err) / bar))
            smax = float(np.max(np.abs(s_ref)))
            assert float(np.max(np.abs(s - s_ref))) <= 1e-11 * smax  # tests/test_spectrum_gpu.py's bar
    finally:
        ref.close()
        dro.close()


# ---------------------------------------------------------------------------------------------- CfarDetector1D
@pytest.fixture(scope="module")
def maps():
    seq = K.map_sequence()
    out = []
    for name, m, delay, doppler, noise in seq:
        out.append(dict(name=name, map=m, delay=delay, doppler=doppler, noise=noise, sq=D.sq_values(m),
                        db_cpu=K.cpu_db(m, noise), db_dev=dev_db(m, delay, doppler, noise)))
    return out


def test_device_db_values_within_the_libm_bound(maps):
    for c in maps:
        assert_db_close(c["db_dev"], c["db_cpu"], c["noise"])


def _sq_dev(m):
    return D.sq_values(m, hypot=lambda a, b: torch.hypot(torch.from_numpy(np.ascontiguousarray(a)).cuda(),
                                                        torch.from_numpy(np.ascontiguousarray(b)).cuda()).cpu().numpy())


def _snr_at(c, lst):
    """The reference's dB value and its bound at each detection's cell."""
    row = np.array([D.hz_to_bin(c["doppler"], f) for f in lst[1]], dtype=np.int64)
    col = (lst[0] - float(c["delay"][0])).astype(np.int64)
    return c["db_cpu"][row, col]


@pytest.mark.parametrize("params", K.CFAR_PARAMS, ids=K.CFAR_IDS)
def test_cfar_object_over_maps_of_changing_shape(maps, params):
    ref, dro = _both(DC.CfarClass, *params)
    try:
        for c in maps:
            a = ref.process(c["map"], c["delay"], c["doppler"], c["noise"])
            b = dro.process(c["map"], c["delay"], c["doppler"], c["noise"])
            assert np.array_equal(b[0], a[0]) and np.array_equal(b[1], a[1]), c["name"]
            want = D.cfar(_sq_dev(c["map"]), c["db_dev"], c["delay"], c["doppler"], *params)
            assert same(b, want), c["name"]
            assert same(a, D.cfar(c["sq"], c["db_cpu"], c["delay"], c["doppler"], *params)), c["name"]
            if len(a[0]):
                ref_db = _snr_at(c, a)
                assert np.all(np.abs(b[2] - a[2]) <= db_bound(ref_db, c["noise"])), c["name"]
    finally:
        ref.close()
        dro.close()


# ---------------------------------------------------------------------------------------------- Centroid
def test_centroid_object_over_lists():
    P = K.CENTROID_P
    ref, dro = _both(DC.CentroidClass, P["nDelay"], P["nDoppler"], P["res"])
    try:
        for name, d, f, s in K.centroid_sequence():
            a = ref.process(d, f, s)
            b = dro.process(d, f, s)
            assert same(b, a), (name, len(a[0]), len(b[0]))
            if d.size <= 4096:
                assert same(a, D.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"])), name
        # past the documented 2^18 detections the drop-in throws rather than truncate the list
        d, f, s = K.clustered_list((1 << 18) + 1)
        with pytest.raises(DC.ClassError, match="capacity"):
            dro.process(d, f, s)
        a = ref.process(d[:100], f[:100], s[:100])  # the object still works afterwards
        assert same(dro.process(d[:100], f[:100], s[:100]), a)
    finally:
        ref.close()
        dro.close()


# ---------------------------------------------------------------------------------------------- Interpolate
def _interp_lists(c):
    """A detection list over map c whose neighbour cells lie inside it (det.cu drops the others on purpose, the
    reference reads outside the map there): Centroid(2, 2, 10) of CFAR(2^-16, 1, 4) on the CPU values, and every
    first / last delay and Doppler cell of the axes."""
    lst = D.centroid(*D.cfar(c["sq"], c["db_cpu"], c["delay"], c["doppler"], D.PFA, 1, 4, -128, 0.0), 2, 2, 10.0)
    d = list(lst[0]) + [float(c["delay"][0]), float(c["delay"][-1])]
    f = list(lst[1]) + [float(c["doppler"][0]), float(c["doppler"][-1])]
    d, f = np.asarray(d), np.asarray(f)
    s = _snr_at(c, (d, f))
    fenced = D.interpolate(d, f, s, c["db_cpu"], c["delay"], c["doppler"], True, True)[3]
    keep = ~fenced
    return d[keep], f[keep], s[keep]


def _parabola_bound(s0, s1, s2, e):
    """|off_dev - off_ref| and |snr_dev - snr_ref| of Interpolate's parabola when every s_k may move by e: with
    num = s0 - s2 and den = 2 (s0 - 2 s1 + s2), off' - off = (dn - off dd) / (den + dd), |dn| <= 2e, |dd| <= 8e; e
    already holds the rounding of each operation (4 ulp of the largest |s_k| on each side)."""
    num, den = s0 - s2, 2 * ((s0 - 2 * s1) + s2)
    off = num / den
    if not math.isfinite(off) or abs(den) <= 8 * e:
        return None
    doff = (2 * e + abs(off) * 8 * e) / (abs(den) - 8 * e)
    dsnr = e + (2 * e * abs(off) + (abs(num) + 2 * e) * doff) / 4
    return doff + 2 * math.ulp(abs(off)), dsnr


def _interp_bounds(c, i, lst, flags):
    """(delay, Doppler, SNR) bounds on the distance between the device's and the reference's output for detection i,
    or None where a parabola is too flat to bound."""
    db, dl, dp = c["db_cpu"], c["delay"], c["doppler"]
    e_of = lambda *v: float(np.max(db_bound(np.array(v), c["noise"]))) + 8 * math.ulp(max(abs(x) for x in v))
    res = float(dp[1] - dp[0])
    d, f, s = float(lst[0][i]), float(lst[1][i]), float(lst[2][i])
    row, col = D.hz_to_bin(dp, f), int(d - float(dl[0]))
    bd = bf = 0.0
    bs = e_of(s)
    if flags[0]:
        b = _parabola_bound(db[row, col - 1], db[row, col], db[row, col + 1], e_of(*db[row, col - 1:col + 2]))
        if b is None:
            return None
        bd, bs = b[0] + math.ulp(abs(d) + 1), max(bs, b[1])
    if flags[1]:
        b = _parabola_bound(db[row - 1, col], db[row, col], db[row + 1, col], e_of(*db[row - 1:row + 2, col]))
        if b is None:
            return None
        bf, bs = abs(res) * b[0] + 2 * math.ulp(abs(f) + abs(res)), max(bs, b[1])
    return bd, bf, bs


def _near_tie(c, i, lst, flags):
    """Whether detection i's peak test (s1 < s0 or s1 < s2 drops it) compares dB values within twice db_bound of
    each other: there the two libraries may decide differently."""
    db, dl, dp = c["db_cpu"], c["delay"], c["doppler"]
    row, col = D.hz_to_bin(dp, float(lst[1][i])), int(float(lst[0][i]) - float(dl[0]))
    trip = []
    if flags[0] and 0 < col < db.shape[1] - 1:
        trip.append(db[row, col - 1:col + 2])
    if flags[1] and 0 < row < db.shape[0] - 1:
        trip.append(db[row - 1:row + 2, col])
    for s0, s1, s2 in trip:
        e = 2 * float(np.max(db_bound(np.array([s0, s1, s2]), c["noise"])))
        if abs(s1 - s0) <= e or abs(s1 - s2) <= e:
            return True
    return False


@pytest.mark.parametrize("flags", [(True, True), (True, False), (False, True), (False, False)])
def test_interpolate_object_over_maps_of_changing_shape(maps, flags):
    """Both builds equal the restatement on their own dB values bit for bit.  Detection by detection (Interpolate
    treats each on its own), the two keep the same detections except at a peak test within the dB bound, and what
    both keep agrees within the bound carried through the parabola."""
    ref, dro = _both(DC.InterpolateClass, *flags)
    try:
        for c in maps:
            if c["map"].shape[0] < 2 or c["map"].shape[1] < 3:
                continue
            lst = _interp_lists(c)
            a = ref.process(*lst, c["map"], c["delay"], c["doppler"], c["noise"])
            b = dro.process(*lst, c["map"], c["delay"], c["doppler"], c["noise"])
            assert same(b, D.interpolate(*lst, c["db_dev"], c["delay"], c["doppler"], *flags)[:3]), c["name"]
            assert same(a, D.interpolate(*lst, c["db_cpu"], c["delay"], c["doppler"], *flags)[:3]), c["name"]
            for i in range(len(lst[0])):
                one = tuple(v[i:i + 1] for v in lst)
                ra = D.interpolate(*one, c["db_cpu"], c["delay"], c["doppler"], *flags)[:3]
                rb = D.interpolate(*one, c["db_dev"], c["delay"], c["doppler"], *flags)[:3]
                if len(ra[0]) != len(rb[0]):
                    assert _near_tie(c, i, lst, flags), (c["name"], i)
                    continue
                bd = _interp_bounds(c, i, lst, flags) if len(ra[0]) else None
                if bd is None:
                    continue
                for j in range(3):
                    if np.isnan(ra[j][0]):
                        assert np.isnan(rb[j][0]), (c["name"], i, j)
                    else:
                        assert abs(rb[j][0] - ra[j][0]) <= bd[j], (c["name"], i, j, rb[j][0], ra[j][0], bd[j])
    finally:
        ref.close()
        dro.close()


# ---------------------------------------------------------------------------------------------- Ambiguity + WienerHopf
def _map_close(got, want):
    mx = float(np.max(np.abs(want)))
    if mx == 0:
        assert float(np.max(np.abs(got))) == 0
        return
    assert float(np.max(np.abs(got - want))) / mx < 1e-5
    assert float(np.linalg.norm(got - want)) / float(np.linalg.norm(want)) < 1e-5


@pytest.mark.parametrize("clutter", [True, False], ids=["clutter", "no_clutter"])
@pytest.mark.parametrize("window", sorted(K.PAIR_GEOMS))
def test_ambiguity_and_wienerhopf_over_consecutive_cpis(window, clutter):
    geom = K.PAIR_GEOMS[window]
    g = O.ambiguity_geometry(*geom)
    args = geom + (K.PAIR_CLUTTER if clutter else None, K.PAIR_FIFO)
    ref, dro = _both(DC.PairClass, *args)
    shape = (g.nDopplerBins, g.nDelayBins)
    try:
        assert dro.n_samples() == ref.n_samples() == g.n
        for k, (x, y) in enumerate(K.pair_pushes(g.n_used, g.n)):
            for o in (ref, dro):
                o.push(x, y)
            if clutter:
                before = [o.fifo(1) for o in (ref, dro)]
                ok = [o.filter() for o in (ref, dro)]
                assert ok[0] == ok[1] == (k != K.PAIR_FAIL_AT), k
                if not ok[0]:  # the failed solve leaves y as it was
                    assert np.array_equal(ref.fifo(1), before[0]) and np.array_equal(dro.fifo(1), before[1])
            _map_close(dro.ambiguity(shape), ref.ambiguity(shape))
            assert dro.n_samples() == ref.n_samples() == g.n_used, k
            xa, xb = ref.fifo(0), dro.fifo(0)
            assert xb.size == xa.size and np.array_equal(xb, xa), k   # leftovers rotated with the same phases
            ya, yb = ref.fifo(1), dro.fifo(1)
            assert yb.size == ya.size, k
            if clutter:
                scale = float(np.max(np.abs(ya)))
                assert float(np.max(np.abs(yb - ya))) <= 1e-9 * scale, k
            else:
                assert np.array_equal(yb, ya), k
    finally:
        ref.close()
        dro.close()


# ---------------------------------------------------------------------------------------------- blah2.cpp loop body
@pytest.fixture(scope="module")
def dropin_refpath():
    harness = os.path.join(os.path.dirname(R.__file__), "_ref", "libdropin_harness.so")
    if not (os.path.exists(harness) and R.available()):
        pytest.skip("refpath harnesses not built (build() with the blah2 sources)")
    spec = importlib.util.spec_from_file_location("dropin_binding_loop", R.__file__)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.LIB_PATH = harness
    return mod


def test_loop_body_over_25_cpis(dropin_refpath):
    from blah2_b200.scene import make_scene

    fs, n = 200000, 40000
    args = dict(delayMin=-5, delayMax=60, dopplerMin=-500, dopplerMax=500, fs=fs, n=n, roundHamming=True,
                clutter=(-5, 30), pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
    ref, dro = R.Chain(**args), dropin_refpath.Chain(**args)
    from blah2_b200.scene import Target
    try:
        for k in range(25):
            sc = make_scene(n, fs, seed=100 + k, targets=[Target(17 + k % 5, 300.0 - 10 * k, -25.0),
                                                          Target(41, -200.0, -28.0)])
            x = np.zeros(n, np.complex128) if k == K.PAIR_FAIL_AT else sc.x
            a, b = ref.run(x, sc.y), dro.run(x, sc.y)
            assert a["skipped"] == b["skipped"] == (k == K.PAIR_FAIL_AT), k
            if a["skipped"]:
                continue
            _map_close(b["map"], a["map"])
            assert abs(b["noisePower"] - a["noisePower"]) < 1e-3, k
            assert len(b["detections"][0]) == len(a["detections"][0]) >= 2, k
            for u, v in zip(b["detections"], a["detections"]):
                assert np.max(np.abs(u - v)) < 1e-2, k
    finally:
        ref.close()
        dro.close()
