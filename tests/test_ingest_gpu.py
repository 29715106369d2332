"""GPU: the int8 (HackRF, Kraken) and complex float32 (USRP) host entry points, with every stage of the chain on.

b200dd_pipeline_submit_host_ci8 equals the int16 entry on the same values bit for bit, in every product; rtl-sdr bytes
are read as int8 as blah2's Kraken source reads them; b200dd_pipeline_submit_host_cf32 equals the device entry on the
same complex64 samples bit for bit and the complex128 entry to FP32 accuracy.  Odd lengths, misaligned and pinned host
buffers, a wrong count, a failed clutter-filter solve and a share set behave as on the other entries."""
import json

import numpy as np
import pytest

import bench
from blah2_b200 import capi
from blah2_b200.process import Pipeline
from blah2_b200.scene import Target, make_scene
from cpi_products import code, cpi_products

pytestmark = pytest.mark.gpu

FS, N = 200000, 40000
SMALL = (-5, 60, -500, 500, FS)
DET = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
DET_DIRECT = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=-5, minDoppler=0.0, nCentroid=4)
TRK = dict(M=2, N=3, delete=4, maxAcc=30, fc=204640000)
METRICS = (0.0, -1.005, 1e21)
T0 = 1731000000000
CFG2 = (bench.GEOM["delayMin"], bench.GEOM["delayMax"], bench.GEOM["dopplerMin"], bench.GEOM["dopplerMax"], bench.FS,
        bench.N)
CFG3 = (0, 511, -256, 256, 10000000, 20000000)  # blah2's 10 MS/s capture, 2 s CPI


def _pipeline(geom, clutter, det):
    """Every stage on: spectrum, clutter filter (unless None), detection, map / detection / IQ-data documents,
    max-hold, tracker and timing."""
    p = Pipeline(*geom, roundHamming=True, clutter=clutter, detection=det, device=0, spectrum_bandwidth=2000,
                 map_json=True, maxhold=True, detection_json=True, max_held_detections=1 << 16, tracker=TRK,
                 max_tracks=1 << 16, max_track_history=32)  # 2 s CPIs at 10 MS/s: 241 hypotheses per detection
    p.enable_iqdata_json(*METRICS)
    p.enable_timing_json(T0)
    return p


def _int8_scene(n, fs, seed, targets, roll=0):
    """A scene quantised to int8: reference power 3600 (I and Q at 42 rms), receiver noise at 1."""
    sc = make_scene(n, fs, seed=seed, targets=targets, sigma_ref=60.0, sigma_noise=1.0, quantise=False)

    def q(z):
        return np.clip(np.round(z.real), -128, 127) + 1j * np.clip(np.round(z.imag), -128, 127)
    return np.roll(q(sc.x), roll), np.roll(q(sc.y), roll)


def _ci8(z):
    b = np.empty((z.shape[0], 2), dtype=np.int8)
    b[:, 0], b[:, 1] = z.real, z.imag
    return b


def _int16(x, y):
    iq = np.empty((x.shape[0], 4), dtype="<i2")
    iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = x.real, x.imag, y.real, y.imag
    return iq


def _timing_shape(doc):
    """A timing document without its stage times, which come from the clock: its keys in order and the values
    that do not (timestamp, nCpi, uptime)."""
    if not isinstance(doc, bytes):
        return doc
    d = json.loads(doc)
    return list(d), [d[k] for k in ("timestamp", "nCpi", "uptime_s", "uptime_days")]


def _stash_shape(doc):
    if not isinstance(doc, bytes):
        return doc
    d = json.loads(doc)
    return [(k, len(v) if isinstance(v, list) else v) for k, v in d.items()]


def _products(pipe, ts):
    """cpi_products as a dict, with the detection count, then the timing document's and stash's shapes."""
    rec = dict(cpi_products(pipe, ts))
    rec["n_detections"] = len(rec["fetch"][2]) // 8
    rec["timing"] = _timing_shape(code(lambda: pipe.fetch_timing_json(ts)))
    rec["timing_stash"] = _stash_shape(code(pipe.fetch_timing_stash))
    return rec


class Feeder:
    """Submits one CPI (complex128 arrays x, y) to a pipeline on one entry point, map_out included, and keeps the
    buffers alive until the next submit."""

    def __init__(self, path):
        self.path, self.keep = path, None

    def submit(self, pipe, x, y):
        g = pipe.geometry
        m = np.full((g.n_doppler_bins, g.n_delay_bins), np.nan, dtype=np.complex128)
        if self.path == "ci8":
            bufs = (_ci8(x), _ci8(y))
            pipe.submit_host_ci8(*bufs, map_out=m)
        elif self.path == "int16":
            bufs = (_int16(x, y),)
            pipe.submit_host_rspduo(*bufs, map_out=m)
        elif self.path == "cf32":
            bufs = (x.astype(np.complex64), y.astype(np.complex64))
            pipe.submit_host_cf32(*bufs, map_out=m)
        elif self.path == "c128":
            bufs = (np.ascontiguousarray(x, dtype=np.complex128), np.ascontiguousarray(y, dtype=np.complex128))
            pipe.submit_host(*bufs, map_out=m)
        else:  # device, eager
            import torch
            dx = torch.from_numpy(x.astype(np.complex64)).cuda()
            dy = torch.from_numpy(y.astype(np.complex64)).cuda()
            dm = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
            torch.cuda.synchronize()
            pipe.submit_device(dx, dy, dm)
            bufs = (dx, dy, dm)
        self.keep = (bufs, m)

    def map_out(self):
        bufs, m = self.keep
        if self.path == "device":
            return bufs[2].cpu().numpy().astype(np.complex128)
        return m


def _run(pipe, path, cpis, ts0=0):
    """Each CPI submitted on `path` and all its products fetched, the map as complex128 bytes."""
    feed = Feeder(path)
    out = []
    for k, (x, y) in enumerate(cpis):
        feed.submit(pipe, x, y)
        rec = _products(pipe, T0 + 1000 * (ts0 + k))
        rec["map_out"] = feed.map_out().tobytes()
        out.append(rec)
    return out


def _assert_same(got, ref, what=""):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys()
        for k in r:
            assert g[k] == r[k], f"{what} CPI {i}: {k} differs"


@pytest.mark.parametrize("config", ["cfg2", "cfg3"])
def test_ci8_equals_int16_bit_for_bit(config):
    geom = CFG2 if config == "cfg2" else CFG3
    tg = [Target(37, 55.0, -40.0), Target(92, -103.0, -45.0), Target(151, 78.0, -45.0)]
    x, y = _int8_scene(geom[5], geom[4], 20261017, tg)
    cpis = [(x, y), (np.roll(x, 977), np.roll(y, 977))]
    outs = {}
    for path in ("ci8", "int16"):
        pipe = _pipeline(geom, bench.CLUTTER, bench.DET)
        outs[path] = _run(pipe, path, cpis)
        pipe.close()
    for rec in outs["int16"]:
        assert not rec["fetch"][0] and rec["n_detections"] > 0
        failed = {k: rec[k] for k in ("map", "maxhold", "detection", "iqdata", "track") if not isinstance(rec[k], bytes)}
        assert not failed, failed
        assert rec["timing"][0][:4] == ["timestamp", "nCpi", "uptime_s", "uptime_days"]
    _assert_same(outs["ci8"], outs["int16"], config)


def _kraken_bytes(z):
    """rtl-sdr's sample bytes: offset binary around 127.5."""
    b = np.empty((z.shape[0], 2), dtype=np.uint8)
    b[:, 0] = np.clip(np.round(127.5 + z.real), 0, 255)
    b[:, 1] = np.clip(np.round(127.5 + z.imag), 0, 255)
    return b


@pytest.mark.parametrize("config", ["filtered", "direct"])
def test_kraken_bytes_are_read_as_int8(config):
    """Kraken.cpp:97-112 reads rtl-sdr's unsigned bytes through an int8_t pointer: the ci8 entry given those bytes
    equals the int16 entry given bytes.view(int8), and differs from the same bytes with their offset removed."""
    clutter, det = ((-5, 30), DET) if config == "filtered" else (None, DET_DIRECT)
    sc = make_scene(N, FS, seed=404, targets=[Target(20, 300.0, -10.0), Target(41, -200.0, -12.0)],
                    sigma_ref=60.0, sigma_noise=1.0, quantise=False)
    xb, yb = _kraken_bytes(sc.x), _kraken_bytes(sc.y)
    assert (xb >= 128).mean() > 0.4 and (yb >= 128).mean() > 0.4
    pipes = [_pipeline(SMALL + (N,), clutter, det) for _ in range(3)]
    g = pipes[0].geometry
    maps = [np.full((g.n_doppler_bins, g.n_delay_bins), np.nan, dtype=np.complex128) for _ in range(3)]
    pipes[0].submit_host_ci8(xb, yb, map_out=maps[0])
    a = _products(pipes[0], T0)
    xs, ys = xb.view(np.int8).astype(np.float64), yb.view(np.int8).astype(np.float64)
    iq = _int16(xs[:, 0] + 1j * xs[:, 1], ys[:, 0] + 1j * ys[:, 1])
    pipes[1].submit_host_rspduo(iq, map_out=maps[1])
    b = _products(pipes[1], T0)
    centred = [(v.astype(np.int16) - 128).astype(np.int8) for v in (xb, yb)]
    pipes[2].submit_host_ci8(*centred, map_out=maps[2])
    c = _products(pipes[2], T0)
    for p in pipes:
        p.close()
    assert not a["fetch"][0] and a["n_detections"] > 0 and c["n_detections"] > 0
    a["map_out"], b["map_out"] = maps[0].tobytes(), maps[1].tobytes()
    _assert_same([a], [b], "kraken")
    assert not np.array_equal(maps[0], maps[2]) and a["map"] != c["map"]


def test_cf32_equals_device_path_and_complex128_entry(relerr):
    tg = [Target(37, 55.0, -40.0), Target(92, -103.0, -45.0)]
    sc = make_scene(bench.N, bench.FS, seed=1017, targets=tg, quantise=False)
    x, y = sc.x.astype(np.complex64), sc.y.astype(np.complex64)
    assert np.any(x.real != np.round(x.real))  # not integers
    cpis = [(x.astype(np.complex128), y.astype(np.complex128))]
    outs = {}
    for path in ("cf32", "device", "c128"):
        pipe = _pipeline(CFG2, bench.CLUTTER, bench.DET)
        outs[path] = _run(pipe, path, cpis)[0]
        pipe.close()
    f, d, h = outs["cf32"], outs["device"], outs["c128"]
    assert not f["fetch"][0] and f["n_detections"] > 0
    _assert_same([f], [d], "cf32 against device")
    # the complex128 entry filters in FP64: the assertions test_rspduo_int16_ingest_matches_complex128_entry makes
    m, hm = np.frombuffer(f["map_out"], np.complex128), np.frombuffer(h["map_out"], np.complex128)
    assert relerr(m, hm)[0] < 1e-5
    assert f["n_detections"] == h["n_detections"]
    fd, hd = np.frombuffer(f["fetch"][2]), np.frombuffer(h["fetch"][2])
    assert np.max(np.abs(fd - hd)) < 1e-3


def _placed(data, pinned, mod, rem):
    """A copy of `data` in host memory at an address = rem (mod `mod`), pageable or pinned."""
    import torch
    raw = torch.empty(data.nbytes + 64, dtype=torch.uint8)
    raw = (raw.pin_memory() if pinned else raw).numpy()
    off = (rem - raw.ctypes.data) % mod
    v = raw[off:off + data.nbytes].view(data.dtype).reshape(data.shape)
    v[...] = data
    assert v.ctypes.data % mod == rem
    return v, raw


# (N, clutter): N odd and N = 2 or 3 (mod 4), filtered; and unfiltered at N = 40001, where the spectrum's nfft
# (40000) exceeds the CAF's n_used (39999)
LENGTHS = [(40001, (-5, 30)), (40002, (-5, 30)), (40003, (-5, 30)), (40001, None)]


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("n,clutter", LENGTHS)
def test_lengths_and_host_addresses(n, clutter, pinned):
    det = DET if clutter else DET_DIRECT
    geom = SMALL + (n,)
    tg = [Target(20, 300.0, -20.0), Target(41, -200.0, -22.0)]
    x, y = _int8_scene(n, FS, 55 + n, tg)
    probe = _pipeline(geom, clutter, det)
    if clutter is None:
        sg, _ = capi.spectrum_plan(n, 2000.0)
        assert sg.nfft > probe.geometry.n_used
    probe.close()
    ref = {}
    for path in ("int16", "device"):
        pipe = _pipeline(geom, clutter, det)
        ref[path] = _run(pipe, path, [(x, y)])[0]
        pipe.close()
    assert not ref["int16"]["fetch"][0] and ref["int16"]["n_detections"] > 0
    g = ref["int16"]
    shape = None
    for fmt in ("ci8", "cf32"):
        pipe = _pipeline(geom, clutter, det)
        shape = (pipe.geometry.n_doppler_bins, pipe.geometry.n_delay_bins)
        m = np.full(shape, np.nan, dtype=np.complex128)
        if fmt == "ci8":  # odd byte addresses
            (xb, kx), (yb, ky) = _placed(_ci8(x), pinned, 2, 1), _placed(_ci8(y), pinned, 2, 1)
            pipe.submit_host_ci8(xb, yb, map_out=m)
            want = g
        else:  # 4 (mod 8)
            (xb, kx), (yb, ky) = (_placed(v.astype(np.complex64), pinned, 8, 4) for v in (x, y))
            pipe.submit_host_cf32(xb, yb, map_out=m)
            want = ref["device"]
        rec = _products(pipe, T0)
        rec["map_out"] = m.tobytes()
        pipe.close()
        _assert_same([rec], [want], f"{fmt} n={n}")
        assert np.array_equal(m, np.frombuffer(g["map_out"], np.complex128).reshape(shape))


def test_wrong_count_enqueues_nothing_and_keeps_the_last_cpi():
    geom = SMALL + (N,)
    tg = [Target(20, 300.0, -20.0)]
    x, y = _int8_scene(N, FS, 77, tg)
    pipe = _pipeline(geom, (-5, 30), DET)
    ref = _run(_pipeline(geom, (-5, 30), DET), "int16", [(x, y)])[0]
    g = pipe.geometry
    m = np.full((g.n_doppler_bins, g.n_delay_bins), np.nan, dtype=np.complex128)
    bx, by = _ci8(x), _ci8(y)
    pipe.submit_host_ci8(bx, by, map_out=m)
    untouched = np.full_like(m, 7.0)
    for f in (lambda: pipe.submit_host_ci8(bx[:-1], by[:-1], map_out=untouched),
              lambda: pipe.submit_host_ci8(np.concatenate([bx, bx[:1]]), np.concatenate([by, by[:1]]),
                                           map_out=untouched),
              lambda: pipe.submit_host_cf32(x[:-1].astype(np.complex64), y[:-1].astype(np.complex64),
                                            map_out=untouched)):
        with pytest.raises(capi.B200ddError) as e:
            f()
        assert e.value.code == capi.ERR_ARG and b"wrong number of samples" in str(e.value).encode()
    rec = _products(pipe, T0)
    rec["map_out"] = m.tobytes()
    _assert_same([rec], [ref], "after refused submits")
    assert np.all(untouched == 7.0)
    pipe.close()


@pytest.mark.parametrize("fmt", ["ci8", "cf32"])
def test_zero_reference_channel_skips_the_cpi(fmt):
    geom = SMALL + (N,)
    x, y = _int8_scene(N, FS, 91, [Target(20, 300.0, -20.0)])
    bad = (np.zeros_like(x), y)
    ref_path = "int16" if fmt == "ci8" else "device"
    pipe = _pipeline(geom, (-5, 30), DET)
    refp = _pipeline(geom, (-5, 30), DET)
    got = _run(pipe, fmt, [bad, (x, y)])
    ref = _run(refp, ref_path, [bad, (x, y)])
    pipe.close()
    refp.close()
    assert got[0]["fetch"][0] and got[0]["n_detections"] == 0
    for k in ("map", "maxhold", "detection", "iqdata", "track", "timing"):
        assert got[0][k] == capi.FILTER_FAILED, k
    assert not got[1]["fetch"][0] and got[1]["n_detections"] > 0
    _assert_same(got, ref, fmt)


def test_share_set_alternated_with_ci8_equals_one_pipeline():
    geom = SMALL + (N,)
    rng = np.random.default_rng(3)
    cpis = []
    for i in range(8):
        tg = [Target(int(rng.integers(8, 55)), float(rng.uniform(-400, 400)), float(rng.uniform(-25, -15)))
              for _ in range(2)]
        cpis.append(_int8_scene(N, FS, 900 + i, tg))
    one = _pipeline(geom, (-5, 30), DET)
    ref = _run(one, "ci8", cpis)
    one.close()
    assert all(r["n_detections"] > 0 for r in ref)
    pipes = [_pipeline(geom, (-5, 30), DET) for _ in range(3)]
    Pipeline.share_history(pipes)
    feeds = [Feeder("ci8") for _ in pipes]
    out = [None] * len(cpis)
    P = len(pipes)

    def products(j):
        rec = _products(pipes[j % P], T0 + 1000 * j)
        rec["map_out"] = feeds[j % P].map_out().tobytes()
        out[j] = rec
    for k, (x, y) in enumerate(cpis):
        feeds[k % P].submit(pipes[k % P], x, y)
        if k - P + 1 >= 0:
            products(k - P + 1)
    for j in range(len(cpis) - P + 1, len(cpis)):
        products(j)
    for p in pipes:
        p.close()
    _assert_same(out, ref, "share set")
