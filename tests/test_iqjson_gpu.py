"""GPU: the IQ-data document and the /stash/iqdata history rendered on the device are blah2's, byte for byte: the
stand-alone handle against tests/golden/iqdata_docs.npz and the host render, the history after every document against
tests/golden/iqdata_stash.npz and oracle/stash_iqdata.py run live, the error codes, and the pipeline stage against the
host render of the spectrum the pipeline returned, on every submit path."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import IqDataJson, Pipeline
from blah2_b200.scene import Target, make_scene
from iqjson_spectra import full_spectrum
from oracle.stash_iqdata import N_CPI, Stash

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DOCS = np.load(os.path.join(GOLD, "iqdata_docs.npz"))
STASH = np.load(os.path.join(GOLD, "iqdata_stash.npz"))
NAMES = sorted(k[:-4] for k in DOCS.files if k.endswith("_doc"))
TS_MAX = 18446744073709551615


def _dev(s):
    import torch
    return torch.from_numpy(np.ascontiguousarray(s, dtype=np.complex128)).cuda()


def _fetch(ij, ts):
    """(status, document) of b200dd_iqjson_fetch."""
    n = C.c_size_t()
    rc = capi.load().b200dd_iqjson_fetch(ij._h, int(ts), capi.ptr(ij._out), ij._out.size, C.byref(n), None)
    return rc, ij._out[:n.value].tobytes()


def _body(doc):
    i = doc.index(b'"spectrum":[') + 12
    return doc[:i], doc[i:-2].split(b",")


def _boundary_diffs(dev_doc, ref_doc, values):
    """Number of spectrum entries where the device document differs from the reference's.  Each such entry must be
    the text of the device's own double, and the reference's text that of a double within two ulp of it: CUDA's
    log10 / hypot and glibc's differed in the last bit there, next to a 0.01 boundary."""
    if dev_doc == ref_doc:
        return 0
    hd, bd = _body(dev_doc)
    hr, br = _body(ref_doc)
    assert hd == hr and len(bd) == len(br) == values.size
    bad = [j for j in range(values.size) if bd[j] != br[j]]
    for j in bad:
        v = values[j]
        near = [v, np.nextafter(v, -np.inf), np.nextafter(np.nextafter(v, -np.inf), -np.inf), np.nextafter(v, np.inf),
                np.nextafter(np.nextafter(v, np.inf), np.inf)]
        texts = [t.encode() for t in capi.format_track_doubles(near)]
        assert bd[j] == texts[0] and br[j] in texts[1:], (j, v, bd[j], br[j])
    return len(bad)


def _device_doc(ij, s, ts):
    """Renders s on the device; (status, document, the device's bin doubles)."""
    d = _dev(s)
    values = ij.bin_values(d)
    ij.render_device(d)
    rc, doc = _fetch(ij, ts)
    return rc, doc, values


@pytest.mark.parametrize("name", NAMES)
def test_device_render_equals_the_stored_reference_documents(name):
    s, m, ts = DOCS[name + "_spectrum"], tuple(DOCS[name + "_metrics"]), int(DOCS[name + "_ts"])
    doc, ok = DOCS[name + "_doc"].tobytes(), bool(DOCS[name + "_ok"])
    ij = IqDataJson(s.size, *m, device=0)
    rc, got, values = _device_doc(ij, s, ts)
    host_v = 10.0 * np.log10(np.hypot(s.real, s.imag))
    with np.errstate(invalid="ignore"):
        ndiff = int(np.sum((values != host_v) & np.isfinite(host_v)))
    if not ok:
        assert rc == capi.ERR_NONFINITE and got == b""
        assert ij.fetch_stash() == b"[]"  # nothing committed
    else:
        assert rc == capi.OK
        assert got == IqDataJson.render_host(s, *m, ts) or _boundary_diffs(got, IqDataJson.render_host(s, *m, ts), values)
        nb = _boundary_diffs(got, doc, values)
        print(f"{name}: {s.size} bins, {ndiff} bin doubles differ from numpy's, {nb} texts at a 0.01 boundary")
    ij.close()


def test_device_render_of_the_full_spectrum():
    s = full_spectrum()
    ij = IqDataJson(s.size, 0.0, 0.0, 0.0, device=0)
    rc, doc, values = _device_doc(ij, s, TS_MAX)
    assert rc == capi.OK
    host = IqDataJson.render_host(s, 0.0, 0.0, 0.0, TS_MAX)
    assert len(host) == int(DOCS["full_len"]) and hashlib.sha256(host).digest() == DOCS["full_sha256"].tobytes()
    nb = _boundary_diffs(doc, host, values)
    print(f"full: {s.size} bins, {nb} texts at a 0.01 boundary")
    assert len(doc) <= ij.max_bytes
    st = Stash()
    st.push(doc)
    assert ij.fetch_stash() == st.send()
    ij.close()


def test_stash_after_every_document_equals_the_fixture_and_the_restatement():
    ts, spectra, metrics, ok = STASH["ts"], STASH["spectra"], tuple(STASH["metrics"]), STASH["ok"]
    dlen, slen = STASH["doc_len"], STASH["stash_len"]
    docs, sent = STASH["docs"].tobytes(), STASH["stash"].tobytes()
    do, so = np.concatenate([[0], np.cumsum(dlen)]), np.concatenate([[0], np.cumsum(slen)])
    assert ts.size > N_CPI + 5
    ij = IqDataJson(spectra.shape[1], *metrics, device=0)
    assert ij.fetch_stash() == b"[]"
    st = Stash()
    exact = True  # every device document so far equals the stored one
    for i in range(ts.size):
        rc, doc, values = _device_doc(ij, spectra[i], int(ts[i]))
        if not ok[i]:  # the stored text is the reference's truncated one, which the stash rejects
            assert rc == capi.ERR_NONFINITE and doc == b""
        else:
            assert rc == capi.OK
            exact &= _boundary_diffs(doc, docs[do[i]:do[i + 1]], values) == 0
            st.push(doc)
        got = ij.fetch_stash()
        assert got == st.send(), i
        if exact:
            assert got == sent[so[i]:so[i + 1]], i
        assert len(got) <= ij.stash_max_bytes
    assert exact, "a device text sat at a 0.01 boundary: the fixture comparison stopped there"
    ij.close()


def test_error_codes_and_misuse():
    lib = capi.load()
    h = C.c_void_p()
    for n, m in ((0, (0.0, 0.0, 0.0)), (65537, (0.0, 0.0, 0.0)), (8, (np.nan, 0.0, 0.0)), (8, (0.0, np.inf, 0.0)),
                 (8, (0.0, 0.0, -np.inf))):
        assert lib.b200dd_iqjson_create(n, *m, 0, C.byref(h)) == capi.ERR_ARG and not h.value
    ij = IqDataJson(65536, 1.0, 2.0, 3.0, device=0)
    with pytest.raises(capi.B200ddError) as e:  # nothing rendered
        ij.fetch(1)
    assert e.value.code == capi.ERR_ARG
    s = full_spectrum()
    rc, doc, _ = _device_doc(ij, s, 1)
    assert rc == capi.OK
    first = ij.fetch_stash()
    s2 = s.copy()
    s2[65535] = 0.0  # a zero last bin: no document, nothing committed
    rc, doc2, _ = _device_doc(ij, s2, 2)
    assert rc == capi.ERR_NONFINITE and doc2 == b""
    assert ij.fetch_stash() == first
    with pytest.raises(capi.B200ddError) as e:  # the rejected render was consumed
        ij.fetch(2)
    assert e.value.code == capi.ERR_ARG
    d = _dev(s[::-1])
    ij.render_device(d)
    out = np.empty(64, dtype=np.uint8)
    n = C.c_size_t()
    rc = lib.b200dd_iqjson_fetch(ij._h, 3, capi.ptr(out), out.size, C.byref(n), None)
    assert rc == capi.ERR_CAPACITY and n.value > 64
    assert ij.fetch_stash() == first  # a too-small buffer commits nothing ...
    doc3 = ij.fetch(3)  # ... and leaves the render to fetch again
    assert doc3.startswith(b'{"timestamp":3,"min":1.0,"max":2.0,"mean":3.0,"frequency":[],"spectrum":[')
    st = Stash()
    st.push(doc)
    st.push(doc3)
    assert ij.fetch_stash() == st.send()
    rc = lib.b200dd_iqjson_fetch_stash(ij._h, capi.ptr(out), out.size, C.byref(n), None)
    assert rc == capi.ERR_CAPACITY and n.value == len(st.send())
    ij.close()


# ---- the pipeline stage, on every submit path

FS, N = 200000, 40000
DET = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
N_PIPE = 24
ZERO_REF = 9  # the CPI whose reference channel is zero: its solve fails
METRICS = (0.0, -1.005, 1e21)


def _pipeline(iqdata=True, **kw):
    p = Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, clutter=(-5, 30), detection=DET, device=0,
                 spectrum_bandwidth=2000, **kw)
    if iqdata:
        p.enable_iqdata_json(*METRICS)
    return p


def _scenes(n=N_PIPE):
    rng = np.random.default_rng(6)
    out = []
    for i in range(n):
        tg = [Target(int(rng.integers(8, 55)), float(rng.uniform(-400, 400)), float(rng.uniform(-35, -20)))
              for _ in range(int(rng.integers(1, 4)))]
        sc = make_scene(N, FS, seed=500 + i, targets=tg)
        out.append((np.zeros_like(sc.x) if i == ZERO_REF else sc.x, sc.y))
    return out


@pytest.mark.parametrize("path", ["process_host", "submit_host", "submit_host_rspduo", "device_eager", "device_graph"])
def test_pipeline_stage_on_every_submit_path(path):
    import torch
    pipe = _pipeline()
    assert pipe.n_spectrum == 2000
    assert pipe.fetch_iqdata_stash() == b"[]"
    g = pipe.geometry
    dx = torch.empty(N, dtype=torch.complex64, device="cuda")
    dy = torch.empty_like(dx)
    dmap = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    st = Stash()
    ij = IqDataJson(2000, *METRICS, device=0)  # the stand-alone render of the same bins
    nb = 0
    for i, (x, y) in enumerate(_scenes()):
        if path == "process_host":
            r = pipe.process(x, y)
        else:
            if path == "submit_host":
                pipe.submit_host(x, y)
            elif path == "submit_host_rspduo":  # the scene's samples are integers
                iq = np.empty((N, 4), dtype="<i2")
                iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = x.real, x.imag, y.real, y.imag
                pipe.submit_host_rspduo(iq)
            else:
                dx.copy_(torch.from_numpy(x.astype(np.complex64)))
                dy.copy_(torch.from_numpy(y.astype(np.complex64)))
                torch.cuda.synchronize()
                if path == "device_graph" and i == 0:
                    pipe.prepare_device(dx, dy, dmap)
                else:
                    pipe.submit_device(dx, dy, dmap)
            r = pipe.fetch()
        ts = 1731000000000 + 100 * i
        if i == ZERO_REF:
            assert r["skipped"]
            with pytest.raises(capi.B200ddError) as e:
                pipe.fetch_iqdata_json(ts)
            assert e.value.code == capi.FILTER_FAILED
            assert pipe.fetch_iqdata_stash() == st.send()
            continue
        s = pipe.fetch_spectrum()
        doc = pipe.fetch_iqdata_json(ts)
        rc, alone, values = _device_doc(ij, s, ts)
        assert rc == capi.OK and doc == alone, i
        nb += _boundary_diffs(doc, IqDataJson.render_host(s, *METRICS, ts), values)
        st.push(doc)
        assert pipe.fetch_iqdata_stash() == st.send(), i
    print(f"{path}: {nb} texts at a 0.01 boundary")
    assert len(st.spectrum) == N_CPI
    ij.close()
    pipe.close()


def test_pipeline_stage_needs_the_spectrum_and_is_dropped_with_it():
    p = Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, device=0)
    with pytest.raises(capi.B200ddError) as e:
        p.enable_iqdata_json(*METRICS)
    assert e.value.code == capi.ERR_ARG
    p.close()
    p = _pipeline()
    with pytest.raises(capi.B200ddError) as e:
        p.enable_iqdata_json(np.nan, 0.0, 0.0)
    assert e.value.code == capi.ERR_ARG
    with pytest.raises(capi.B200ddError) as e:  # the failed enable left no stage
        p.fetch_iqdata_stash()
    assert e.value.code == capi.ERR_ARG
    p.enable_iqdata_json(*METRICS)
    x, y = _scenes(1)[0]
    p.process(x, y)
    p.fetch_iqdata_json(1)
    assert capi.load().b200dd_pipeline_enable_spectrum(p._h, 4000.0, None) == capi.OK  # 1000 bins now
    with pytest.raises(capi.B200ddError) as e:
        p.fetch_iqdata_stash()
    assert e.value.code == capi.ERR_ARG
    p.close()


def test_pipeline_stage_changes_no_other_output():
    import torch
    a, b = _pipeline(map_json=True), _pipeline(iqdata=False, map_json=True)
    g = a.geometry
    dx = torch.empty(N, dtype=torch.complex64, device="cuda")
    dy = torch.empty_like(dx)
    maps = [torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda") for _ in range(2)]
    for i, (x, y) in enumerate(_scenes(6)):
        if i < 3:
            ra, rb = a.process(x, y), b.process(x, y)
            assert np.array_equal(ra["map"], rb["map"])
        else:  # graph-replayed
            dx.copy_(torch.from_numpy(x.astype(np.complex64)))
            dy.copy_(torch.from_numpy(y.astype(np.complex64)))
            torch.cuda.synchronize()
            for p, m in ((a, maps[0]), (b, maps[1])):
                (p.prepare_device if i == 3 else p.submit_device)(dx, dy, m)
            ra, rb = a.fetch(), b.fetch()
            assert torch.equal(maps[0], maps[1])
        assert ra["skipped"] == rb["skipped"]
        assert ra["noisePower"] == rb["noisePower"] and ra["maxPower"] == rb["maxPower"]
        da, db = ra["detections"], rb["detections"]
        assert np.array_equal(da.delay, db.delay) and np.array_equal(da.doppler, db.doppler)
        assert np.array_equal(da.snr, db.snr)
        assert np.array_equal(a.fetch_spectrum(), b.fetch_spectrum())
        if not ra["skipped"]:
            assert a.fetch_map_json(i) == b.fetch_map_json(i)
    a.close()
    b.close()
