"""GPU: the map document of blah2.cpp:303-304 (delay_bin_to_km(to_json(ts), fs)) rendered on the device is the
reference's, byte for byte: the device formatter against the host one, the stand-alone renders against the
reference's documents of tests/golden/map_json_maps.npz, and the pipeline stage against the stand-alone render of
the map and metrics the same CPI produced."""
import hashlib
import os

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import Map, MapJson, Pipeline
from blah2_b200.scene import Target, make_scene
from map_json_maps import MAPS, hash_map, k_grid

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def test_device_formatter_equals_host_formatter():
    z = gold("map_json_values")
    rng = np.random.default_rng(11)
    sets = [k_grid()[1].ravel(), z["small"], z["bits"].view(np.float64),
            rng.integers(0, 2 ** 64, 1 << 24, dtype=np.uint64).view(np.float64)]
    for vals in sets:
        host = capi.format_doubles(vals)
        dev = capi.format_doubles(vals, device=0)
        if host != dev:
            bad = [(vals[i], dev[i], host[i]) for i in range(vals.size) if dev[i] != host[i]]
            pytest.fail(f"{len(bad)} of {vals.size} differ: {bad[:5]}")


def _check_doc(name, doc):
    z = gold("map_json_maps")
    if MAPS[name].get("full"):
        assert doc == z[name + "_doc"].tobytes()
    assert len(doc) == int(z[name + "_len"])
    assert hashlib.sha256(doc).digest() == z[name + "_sha256"].tobytes()


@pytest.mark.parametrize("name", list(MAPS))
def test_renders_equal_the_reference(name):
    import torch
    spec = MAPS[name]
    m, delay, doppler = hash_map(spec)
    noise, maxp = (float(v) for v in gold("map_json_maps")[name + "_metrics"])
    mj = MapJson(delay, doppler, spec["fs"], device=0)
    assert mj.max_bytes >= int(gold("map_json_maps")[name + "_len"])
    d64 = torch.from_numpy(m).cuda()
    d32 = d64.to(torch.complex64)  # the map holds float32 values: widening gives the same doubles
    # how many cell doubles differ from the host libm (CUDA's log10 / hypot against glibc's): reported only; the
    # document must be identical all the same unless one sits within an ulp of a 0.01 boundary
    host_v = 10.0 * np.log10(np.hypot(m.real, m.imag)) - noise
    ndiff = int(np.sum(mj.cell_values(d64, noise) != host_v))
    print(f"{name}: {m.size} cells, {ndiff} cell doubles differ from numpy's")
    _check_doc(name, Map(m, delay, doppler, noise, maxp).to_json_km(spec["ts"], spec["fs"], device=0))
    _check_doc(name, mj.render_host(m, noise, maxp, spec["ts"]))
    for d in (d64, d32):
        mj.render_device(d, noise, maxp)
        _check_doc(name, mj.fetch(spec["ts"]))
    mj.close()


def test_misuse_and_non_finite_cells():
    import torch
    spec = MAPS["small"]
    m, delay, doppler = hash_map(spec)
    mj = MapJson(delay, doppler, spec["fs"], device=0)
    for bad in (0.0, np.nan, np.inf):
        mm = m.copy()
        mm[5, 7] = bad
        with pytest.raises(capi.B200ddError) as e:
            mj.render_host(mm, 60.0, 300.0, 1)
        assert e.value.code == capi.ERR_NONFINITE
    with pytest.raises(capi.B200ddError) as e:  # a non-finite noisePower makes every cell non-finite
        mj.render_host(m, np.nan, 300.0, 1)
    assert e.value.code == capi.ERR_NONFINITE
    # a good map on the same handle afterwards
    assert mj.render_host(m, 60.0, 300.0, 1).startswith(b'{"timestamp":1,"nRows":17,"nCols":33,"noisePower":60.0,')
    d = torch.from_numpy(m).cuda()
    mj.render_device(d, 60.0, 300.0)
    out = np.empty(16, dtype=np.uint8)
    import ctypes as C
    n = C.c_size_t()
    rc = capi.load().b200dd_mapjson_fetch(mj._h, 1, capi.ptr(out), out.size, C.byref(n), None)
    assert rc == capi.ERR_CAPACITY and n.value > 16
    mj.close()


def _scene_pipeline(**kw):
    fs, n = 200000, 40000
    det = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
    sc = make_scene(n, fs, seed=11, targets=[Target(17, 300.0, -25.0), Target(41, -200.0, -28.0)])
    pipe = Pipeline(-5, 60, -500, 500, fs, n, roundHamming=True, clutter=(-5, 30), detection=det, device=0, **kw)
    return pipe, sc, fs


def _expected(pipe, fs, map_c, res, ts):
    """The stand-alone device render of the map and metrics this CPI produced."""
    mj = MapJson(pipe.delay, pipe.doppler, fs, device=0)
    mj.render_device(map_c, res["noisePower"], res["maxPower"])
    doc = mj.fetch(ts)
    mj.close()
    return doc


def test_pipeline_stage_on_every_submit_path():
    import torch
    pipe, sc, fs = _scene_pipeline(map_json=True)
    assert pipe.map_json_max_bytes > 0
    g = pipe.geometry
    ts = 1731000000000
    # host entry (complex128)
    m = np.empty((g.n_doppler_bins, g.n_delay_bins), dtype=np.complex128)
    pipe.submit_host(sc.x, sc.y, map_out=m)
    r = pipe.fetch()
    assert not r["skipped"]
    doc_host = pipe.fetch_map_json(ts)
    assert doc_host == _expected(pipe, fs, torch.from_numpy(m).cuda(), r, ts)
    assert doc_host.startswith(b'{"timestamp":1731000000000,"nRows":%d,"nCols":%d,' % (g.n_doppler_bins, g.n_delay_bins))
    # rspduo int16 entry (the scene's samples are integers)
    iq = np.empty((sc.x.size, 4), dtype="<i2")
    iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = sc.x.real, sc.x.imag, sc.y.real, sc.y.imag
    m2 = np.empty_like(m)
    pipe.submit_host_rspduo(iq, map_out=m2)
    r2 = pipe.fetch()
    assert pipe.fetch_map_json(ts + 1) == _expected(pipe, fs, torch.from_numpy(m2).cuda(), r2, ts + 1)
    # device entry: eager, then recorded and replayed as a graph, on a caller stream
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    dmap = torch.zeros((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    s = torch.cuda.Stream()
    docs = []
    with torch.cuda.stream(s):
        pipe.submit_device(dx, dy, dmap, s.cuda_stream)
        r3 = pipe.fetch(s.cuda_stream)
        docs.append(pipe.fetch_map_json(ts + 2))
        want = _expected(pipe, fs, dmap.clone(), r3, ts + 2)
        pipe.prepare_device(dx, dy, dmap, s.cuda_stream)
        for _ in range(2):
            dmap.zero_()
            pipe.submit_device(dx, dy, dmap, s.cuda_stream)
            r4 = pipe.fetch(s.cuda_stream)
            docs.append(pipe.fetch_map_json(ts + 2))
    s.synchronize()
    assert docs[0] == want
    assert all(d == want for d in docs[1:]) and r4["noisePower"] == r3["noisePower"]


def test_pipeline_stage_skips_failed_solves_and_leaves_other_pipelines_alone():
    import torch
    n = 8192
    det = dict(pfa=1e-3, nGuard=1, nTrain=4, minDelay=0, minDoppler=0.0, nCentroid=2)
    pipe = Pipeline(-3, 20, -50, 50, 10000, n, clutter=(-2, 10), detection=det, device=0, map_json=True)
    plain = Pipeline(-3, 20, -50, 50, 10000, n, clutter=(-2, 10), detection=det, device=0)
    rng = np.random.default_rng(5)
    y = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 100.0
    out = pipe.process(np.zeros(n, complex), y)  # zero reference channel: the solve fails
    assert out["skipped"]
    with pytest.raises(capi.B200ddError) as e:
        pipe.fetch_map_json(5)
    assert e.value.code == capi.FILTER_FAILED
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 100.0
    a, b = pipe.process(x, 0.5 * x + y * 1e-3), plain.process(x, 0.5 * x + y * 1e-3)
    assert not a["skipped"] and np.array_equal(a["map"], b["map"]) and a["noisePower"] == b["noisePower"]
    doc = pipe.fetch_map_json(6)
    assert doc == _expected(pipe, 10000, torch.from_numpy(a["map"]).cuda(), a, 6)
    with pytest.raises(capi.B200ddError) as e:
        plain.fetch_map_json(6)
    assert e.value.code == capi.ERR_ARG
