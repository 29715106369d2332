"""GPU: CPI records.  Pipelines that export every CPI as a record, standing in for the ranks of the independent-CPI
mode, and an importer that takes the records and maps in CPI order give every product one pipeline gives when it
runs all the CPIs itself: fetch results, maps, every document and stash after every CPI, and the tracker's
documents.  Records agree across submit entries, export changes nothing the exporter computes, and a record of other
parameters or stages is refused."""
import ctypes as C
import json
import struct

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import Pipeline, record_bytes, timing_render_host
from cpi_products import code, cpi_products

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

DET = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
TRK = dict(M=2, N=3, delete=4, maxAcc=30, fc=204640000)
METRICS = (0.0, -1.005, 1e21)
T_START = 1730999990000
N_CPI = 26
BAD = 12   # an all-zero reference channel: the clutter filter's solve fails

# config 2 (BASELINE.md), and the map and CPI size of config 4 with config 2's clutter window
GEOMS = {
    "cfg2": dict(delayMin=0, delayMax=299, dopplerMin=-128, dopplerMax=128, fs=2_000_000, nSamples=2_000_000,
                 clutter=(-10, 400)),
    "cfg4": dict(delayMin=0, delayMax=511, dopplerMin=-512, dopplerMax=512, fs=10_000_000, nSamples=10_000_000,
                 clutter=(-10, 400)),
}


def _ts(i):
    return 1731000000000 + 100 * i


def _pipeline(geom, products=True, timing=True, spectrum=True, export=None, **over):
    g = dict(GEOMS[geom])
    g.update(over)
    kw = dict(roundHamming=True, device=0, detection=DET)
    if spectrum:
        kw["spectrum_bandwidth"] = 2000
    if products:
        kw.update(map_json=True, maxhold=True, detection_json=True, max_held_detections=1 << 16, tracker=TRK,
                  max_tracks=1 << 12, max_track_history=32)
    p = Pipeline(**g, **kw)
    if products and spectrum:
        p.enable_iqdata_json(*METRICS)
    if timing:
        p.enable_timing_json(T_START)
    if export:
        p.enable_export(export)
    return p


_SCENES = {}


def _scenes(geom, n=N_CPI, integer=False):
    """n CPIs of complex64 device samples: a reference channel and echoes of it at a few delays and Doppler shifts
    (generated on the device).  integer: every sample an integer in int8 range (exact in every host format)."""
    key = (geom, n, integer)
    if key not in _SCENES:
        g = GEOMS[geom]
        N, fs = g["nSamples"], g["fs"]
        gen = torch.Generator(device="cuda")
        t = torch.arange(N, device="cuda", dtype=torch.float64) / fs
        out = []
        for i in range(n):
            gen.manual_seed(900 + i)
            x = torch.randn(N, 2, device="cuda", generator=gen).view(torch.complex64).reshape(N) * 10
            y = torch.randn(N, 2, device="cuda", generator=gen).view(torch.complex64).reshape(N) * 3 + 8 * x
            for k in range(1 + i % 3):
                d = int(torch.randint(8, g["delayMax"] - 8, (1,), device="cuda", generator=gen))
                f = (20 + 40 * float(torch.rand(1, device="cuda", generator=gen))) * (1 if k % 2 else -1)
                y = y + 0.3 * torch.roll(x, d) * torch.exp(2j * np.pi * f * t).to(torch.complex64)
            if integer:
                x = torch.complex(x.real.round().clamp(-127, 127), x.imag.round().clamp(-127, 127))
                y = torch.complex(y.real.round().clamp(-127, 127), y.imag.round().clamp(-127, 127))
            if i == BAD and n == N_CPI:
                x = torch.zeros_like(x)
            out.append((x.contiguous(), y.contiguous()))
        torch.cuda.synchronize()
        _SCENES[key] = out
    return _SCENES[key]


def _map_buf(p):
    g = p.geometry
    return torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")


def _raw_fetch(p):
    """b200dd_pipeline_fetch's return code and results (Pipeline.fetch accepts ERR_CAPACITY silently)."""
    res = capi.CpiResult()
    rc = p._lib.b200dd_pipeline_fetch(p._h, C.byref(res), capi.ptr(p._od), capi.ptr(p._of), capi.ptr(p._os), p.cap,
                                      None)
    n = min(res.n_detections, p.cap)
    return (rc, res.filter_status, struct.pack("<2d", res.noise_power, res.max_power), p._od[:n].tobytes(),
            p._of[:n].tobytes(), p._os[:n].tobytes())


def _products(p, i, timing=True):
    """CPI i's fetch and then every product, in blah2's order; the timing document is checked against the stand-alone
    render of its names and values and returned as (names, values) instead of bytes."""
    ts = _ts(i)
    out = cpi_products(p, ts, fetch=_raw_fetch)
    tm = None
    if timing:
        doc = code(lambda: p.fetch_timing_json(ts))
        if isinstance(doc, bytes):
            names, values = p.timing_values()
            n_cpi = json.loads(doc)["nCpi"]
            assert doc == timing_render_host(T_START, ts, n_cpi, names, values)
            tm = dict(zip(names, values))
        else:
            tm = doc
    return out, tm


_REFS = {}


def _reference(geom):
    """One pipeline running every CPI itself (submit_device, eager): its maps and products after every CPI."""
    if geom not in _REFS:
        p = _pipeline(geom)
        m = _map_buf(p)
        maps, prods = [], []
        for i, (x, y) in enumerate(_scenes(geom)):
            p.submit_device(x, y, m)
            torch.cuda.synchronize()
            maps.append(m.clone())
            prods.append(_products(p, i)[0])
        torch.cuda.synchronize()
        _REFS[geom] = (maps, prods)
        p.close()
    return _REFS[geom]


def _export_all(geom, k):
    """K exporting pipelines used round-robin: every CPI's record and map copied out, the exporter's own timing
    values, and afterwards one more CPI on each exporter so that none of its buffers still holds an exported CPI."""
    exps = [_pipeline(geom, products=False, export=4096) for _ in range(k)]
    bufs = [_map_buf(e) for e in exps]
    assert exps[0].record_bytes == record_bytes(4096, exps[0].n_spectrum, timing=True)
    recs, maps, tms = [], [], []
    scenes = _scenes(geom)
    for i, (x, y) in enumerate(scenes):
        e, m = exps[i % k], bufs[i % k]
        e.submit_device(x, y, m)
        torch.cuda.synchronize()
        recs.append(e.export_record().clone())
        maps.append(m.clone())
        torch.cuda.synchronize()
        e.fetch()
        doc = code(lambda: e.fetch_timing_json(_ts(i)))
        tms.append(dict(zip(*e.timing_values())) if isinstance(doc, bytes) else doc)
    for j, e in enumerate(exps):
        x, y = scenes[j]
        e.submit_device(x, y, bufs[j])
        e.fetch()
    torch.cuda.synchronize()
    return exps, recs, maps, tms


def _check_timing(i, got, exported):
    if i == BAD:
        assert got == capi.FILTER_FAILED and exported == capi.FILTER_FAILED
        return
    assert set(got) == set(exported) | {"tracker"}
    for name, v in exported.items():
        if name != "cpi":
            assert got[name] == v, (i, name)
    assert got["cpi"] == exported["cpi"] + got["tracker"]


@pytest.mark.parametrize("geom", ["cfg2", "cfg4"])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_imported_cpis_equal_one_pipeline(geom, k):
    """K exporters (the ranks) and one importer (rank 0), and a share set of importers, against one pipeline that
    ran every CPI: maps, fetch results and every document and stash identical after every CPI, the timing document
    the render of the exporter's stage times plus rank 0's tracker time."""
    ref_maps, ref_prods = _reference(geom)
    exps, recs, maps, tms = _export_all(geom, k)
    for i in range(N_CPI):
        assert torch.equal(maps[i], ref_maps[i]), i
    # one importer
    imp = _pipeline(geom)
    for i in range(N_CPI):
        imp.submit_record(recs[i], maps[i])
        got, tm = _products(imp, i)
        assert got == ref_prods[i], i
        _check_timing(i, tm, tms[i])
    # a share set of importers, each CPI fetched after the next one was imported
    members = [_pipeline(geom) for _ in range(max(k, 2))]
    Pipeline.share_history(members)
    for i in range(N_CPI + 1):
        if i < N_CPI:
            members[i % len(members)].submit_record(recs[i], maps[i])
        if i >= 1:
            got, tm = _products(members[(i - 1) % len(members)], i - 1)
            assert got == ref_prods[i - 1], i - 1
            _check_timing(i - 1, tm, tms[i - 1])
    assert all(r[0][1][1] == capi.OK for j, r in enumerate(ref_prods) if j != BAD)
    assert ref_prods[BAD][0][1][1] == capi.FILTER_FAILED
    assert any(len(r[0][1][3]) for r in ref_prods)   # CPIs with detections


def _mask_path(rec):
    r = rec.clone()
    r[4:8] = 0   # the header's submit-path word: host entries count their copies as extract_buffer
    return r


def test_records_agree_across_submit_entries():
    """Integer samples, exact in every host format: the eager and graph-replayed device chains, the int16, int8 and
    complex64 host entries give one record (but for the path word); the complex128 entry's record imports as the
    exporter's own products."""
    geom = "cfg2"
    scenes = _scenes(geom, n=3, integer=True)
    recs = {}
    for entry in ("device_eager", "device_graph", "rspduo", "ci8", "cf32", "c128"):
        p = _pipeline(geom, products=False, timing=False, export=512)
        m = _map_buf(p)
        out = []
        for i, (x, y) in enumerate(scenes):
            if entry == "device_eager":
                p.submit_device(x, y, m)
            elif entry == "device_graph":
                if i == 0:
                    p.prepare_device(x, y, m)   # an eager CPI, then the graph
                p.submit_device(x, y, m)
            else:
                xh, yh = x.cpu().numpy(), y.cpu().numpy()
                if entry == "rspduo":
                    iq = np.empty((xh.size, 4), dtype="<i2")
                    iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = xh.real, xh.imag, yh.real, yh.imag
                    p.submit_host_rspduo(iq)
                elif entry == "ci8":
                    p.submit_host_ci8(np.stack([xh.real, xh.imag], 1).astype(np.int8),
                                      np.stack([yh.real, yh.imag], 1).astype(np.int8))
                elif entry == "cf32":
                    p.submit_host_cf32(xh, yh)
                else:
                    p.submit_host(xh.astype(np.complex128), yh.astype(np.complex128))
            torch.cuda.synchronize()
            rec = p.export_record().clone()
            mine = _raw_fetch(p)
            if entry == "c128" or entry == "rspduo":
                # the record imports as the exporter's own CPI
                q = _pipeline(geom, products=False, timing=False)
                mm = _map_buf(q)
                if entry == "c128":
                    g = p.geometry
                    mh = np.empty((g.n_doppler_bins, g.n_delay_bins), dtype=np.complex128)
                    p.submit_host(xh.astype(np.complex128), yh.astype(np.complex128), map_out=mh)
                    torch.cuda.synchronize()
                    assert torch.equal(p.export_record(), rec)   # the same CPI again
                    p.fetch()
                    mm.copy_(torch.from_numpy(mh.astype(np.complex64)))
                q.submit_record(rec, mm)   # q renders no map product: the map's content is not read
                assert _raw_fetch(q) == mine
                assert np.array_equal(q.fetch_spectrum(), p.fetch_spectrum())
                q.close()
            out.append(rec)
        recs[entry] = out
        p.close()
    hdr = [struct.unpack("<II", bytes(r[:8].cpu().numpy())) for r in recs["device_eager"]]
    assert all(h[0] == 1 for h in hdr)
    for entry in ("device_graph", "rspduo", "ci8", "cf32"):
        for i in range(len(scenes)):
            assert torch.equal(_mask_path(recs[entry][i]), _mask_path(recs["device_eager"][i])), (entry, i)
    for i in range(len(scenes)):
        assert torch.equal(recs["device_graph"][i], recs["device_eager"][i])


def test_export_changes_nothing_the_exporter_computes():
    """Every stage on, device eager and graph-replayed: with export on, every fetch result, map, document and stash
    of the exporting pipeline is the one the same pipeline gives with export off."""
    geom = "cfg2"
    scenes = _scenes(geom, n=6)
    runs = []
    for export in (None, 4096):
        p = _pipeline(geom, export=export)
        m = _map_buf(p)
        out = []
        for i, (x, y) in enumerate(scenes):
            if i == 3:
                p.prepare_device(x, y, m)
            else:
                p.submit_device(x, y, m)
            torch.cuda.synchronize()
            out.append((m.clone(), _products(p, i)[0], p.timing_values()[0]))
        runs.append(out)
        p.close()
    for (m0, p0, n0), (m1, p1, n1) in zip(*runs):
        assert torch.equal(m0, m1) and p0 == p1 and n0 == n1


def test_failed_solve_imports_as_filter_failed():
    geom = "cfg2"
    scenes = _scenes(geom)
    e = _pipeline(geom, products=False, export=64)
    q = _pipeline(geom)
    m = _map_buf(e)
    stashes = None
    for i in (BAD - 1, BAD, BAD + 1):
        x, y = scenes[i]
        e.submit_device(x, y, m)
        torch.cuda.synchronize()
        q.submit_record(e.export_record().clone(), m.clone())
        got, tm = _products(q, i)
        fetch = got[0][1]
        if i == BAD:
            assert fetch[1] == capi.FILTER_FAILED
            for name, v in got[1:]:
                if name not in ("spectrum", "detection_stash", "iqdata_stash"):
                    assert v == capi.FILTER_FAILED, name
            assert tm == capi.FILTER_FAILED
            assert (got[5][1], got[7][1]) == stashes           # nothing committed
        else:
            assert fetch[1] == capi.OK and isinstance(tm, dict)
            stashes = (got[5][1], got[7][1])
        if i == BAD + 1:
            assert json.loads(q.last_timing_doc)["nCpi"] == 2   # the failed CPI did not step nCpi
        e.fetch()


def test_record_overflow_acts_as_cfar_overflow():
    """Two detection slots: a CPI with more detections imports as a CFAR overflow -- fetch and the detection document
    return ERR_CAPACITY, the detection history and the tracker skip it; metrics, map and spectrum are imported."""
    geom = "cfg2"
    scenes = _scenes(geom)
    ref = _pipeline(geom)
    e = _pipeline(geom, products=False, export=2)
    assert e.record_bytes == record_bytes(2, e.n_spectrum, timing=True)
    q = _pipeline(geom)
    m = _map_buf(e)
    seen = False
    for i in range(6):
        x, y = scenes[i]
        e.submit_device(x, y, m)
        ref.submit_device(x, y)
        torch.cuda.synchronize()
        q.submit_record(e.export_record().clone(), m.clone())
        r = _raw_fetch(ref)
        n = len(r[3]) // 8
        stash0 = q.fetch_detection_stash()
        got, tm = _products(q, i)
        if n <= 2:
            assert got[0][1] == r
            continue
        seen = True
        rc, fs, metrics = got[0][1][:3]
        assert rc == capi.ERR_CAPACITY and fs == capi.OK and metrics == r[2]
        d = dict(got)
        assert d["detection"] == capi.ERR_CAPACITY and d["track"] == capi.ERR_CAPACITY
        assert d["detection_stash"] == stash0
        assert isinstance(d["map"], bytes) and isinstance(d["maxhold"], bytes) and isinstance(d["iqdata"], bytes)
        assert tm["tracker"] == 0.0   # the tracker skipped the CPI
        e.fetch()
    assert seen


def test_mismatched_records_are_refused():
    geom = "cfg2"
    x, y = _scenes(geom)[0]
    q = _pipeline(geom)
    others = [
        _pipeline(geom, products=False, export=64, delayMax=298),       # other geometry
        _pipeline(geom, products=False, export=64, clutter=(-10, 399)),  # other clutter window
        _pipeline(geom, products=False, export=64, timing=False),        # no timing stage
        _pipeline(geom, products=False, export=64, spectrum=False),      # no spectrum stage
    ]
    for e in others:
        m = _map_buf(e)
        e.submit_device(x, y, m)
        torch.cuda.synchronize()
        with pytest.raises(capi.B200ddError) as ei:
            q.submit_record(e.export_record(), m)
        assert ei.value.code == capi.ERR_ARG
    # nothing was taken: the importer has no CPI to fetch
    assert code(lambda: q.fetch_map_json(0)) == capi.ERR_ARG
    # a buffer that is not a record
    junk = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    with pytest.raises(capi.B200ddError):
        q.submit_record(junk, _map_buf(q))
    # export_record before any submit, and without export
    e = _pipeline(geom, products=False, export=64)
    with pytest.raises(capi.B200ddError):
        e.export_record()
    with pytest.raises(capi.B200ddError):
        q.export_record()


def test_comm_gather_world1_then_import():
    """A world-1 communicator gathers (record, map) and the import gives the same documents."""
    from blah2_b200.shard import Comm, IndependentCpiPlan
    try:
        comm = Comm(0, 1, 0)
    except Exception as err:  # noqa: BLE001 -- no usable NCCL here
        pytest.skip(f"no NCCL communicator: {err}")
    geom = "cfg2"
    scenes = _scenes(geom)[:4]
    ref = _pipeline(geom)
    e = _pipeline(geom, products=False, export=4096)
    q = _pipeline(geom)
    m = _map_buf(e)
    s = torch.cuda.Stream()
    plan = IndependentCpiPlan(comm, e.record_bytes, tuple(m.shape), "cuda")
    got = []

    def compute(c):
        x, y = scenes[c]
        torch.cuda.synchronize()
        e.submit_device(x, y, m, stream=s.cuda_stream)
        return e.export_record(), m

    def consume(c, rec, mp):
        q.submit_record(rec, mp)
        got.append(_products(q, c, timing=False)[0])

    plan.run(len(scenes), compute, consume, after=s)
    for c, (x, y) in enumerate(scenes):
        ref.submit_device(x, y)
        assert _products(ref, c, timing=False)[0] == got[c]
    comm.close()
