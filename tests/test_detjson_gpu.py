"""GPU: the detection document and the /stash/detection history rendered on the device are blah2's, byte for byte:
the stand-alone handle against tests/golden/detection_docs.npz and the host render, the history after every
document against tests/golden/detection_stash.npz and oracle/stash_detection.py run live, its capacity limits, and
the pipeline stage against the host render of the detections the pipeline returned, on every submit path."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import DetectionJson, Pipeline
from blah2_b200.scene import Target, make_scene
from detjson_lists import LARGE, N_FULL, large_lists
from oracle import refdetjson
from oracle.stash_detection import Stash

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DOCS = np.load(os.path.join(GOLD, "detection_docs.npz"))
STASH = np.load(os.path.join(GOLD, "detection_stash.npz"))
SMALL = sorted(k[:-4] for k in DOCS.files if k.endswith("_doc"))


def _dev(dl, dp, sn, count=None):
    import torch
    n = len(dl) if count is None else count
    # an empty list still gets one (unread) element: the render takes no null list
    t = [torch.from_numpy(np.ascontiguousarray(a if len(a) else [0.0], dtype=np.float64)).cuda() for a in (dl, dp, sn)]
    return t + [torch.tensor([n], dtype=torch.int32, device="cuda")]


def _render(dj, lists, count=None):
    """Renders the lists on the device; returns the device tensors (kept alive until the fetch)."""
    t = _dev(*lists, count=count)
    dj.render_device(*t)
    return t


def _fetch(dj, ts):
    """(status, document) of b200dd_detjson_fetch, also where the status is an error with the document written."""
    n = C.c_size_t()
    rc = capi.load().b200dd_detjson_fetch(dj._h, int(ts), capi.ptr(dj._out), dj._out.size, C.byref(n), None)
    return rc, dj._out[:n.value].tobytes()


@pytest.mark.parametrize("name", SMALL)
def test_device_render_equals_the_stored_reference_documents(name):
    lists = DOCS[name + "_lists"]
    ts, fs = (int(v) for v in DOCS[name + "_meta"])
    dj = DetectionJson(fs, max_held=8192, device=0)
    t = _render(dj, lists)
    rc, doc = _fetch(dj, ts)
    # a value outside int32 hundredths (the exponent forms, km at fs = 1) keeps the document out of the history
    assert rc in (capi.OK, capi.ERR_ARG)
    assert doc == DOCS[name + "_doc"].tobytes() == DetectionJson.render_host(*lists, ts, fs)
    if name in ("one", "empty", "boundaries", "negative_delay", "cfg2_chain", "chain_a"):
        assert rc == capi.OK
    del t
    dj.close()


@pytest.mark.parametrize("name", list(LARGE))
def test_device_render_of_full_lists(name):
    spec = LARGE[name]
    lists = large_lists(name)
    dj = DetectionJson(spec["fs"], max_held=N_FULL, device=0)
    t = _render(dj, lists)
    rc, doc = _fetch(dj, spec["ts"])
    assert len(doc) == int(DOCS[name + "_len"])
    assert hashlib.sha256(doc).digest() == DOCS[name + "_sha256"].tobytes()
    if name == "bounded_full":  # exactly 2^18 entries, all of them held
        assert rc == capi.OK
        st = Stash()
        st.push(doc)
        assert dj.fetch_stash() == st.send()
    del t
    dj.close()


def test_device_render_equals_host_render_on_random_full_lists():
    rng = np.random.default_rng(17)
    for fs in (2000000, int(rng.integers(1, 1 << 32))):
        v = []
        for _ in range(3):
            bits = rng.integers(0, 1 << 52, N_FULL, dtype=np.uint64) | (rng.integers(1023 - 60, 1023 + 90, N_FULL)
                                                                        .astype(np.uint64) << np.uint64(52))
            v.append(bits.view(np.float64) * rng.choice([-1.0, 1.0], N_FULL))
        dj = DetectionJson(fs, max_held=16, device=0)
        t = _render(dj, v)
        rc, doc = _fetch(dj, 1731000000000)
        assert rc in (capi.OK, capi.ERR_ARG, capi.ERR_CAPACITY)
        assert doc == DetectionJson.render_host(*v, 1731000000000, fs)
        del t
        dj.close()


@pytest.mark.parametrize("name", ["quirk", "above_2e53"])
def test_stash_after_every_document_equals_the_fixture_and_the_restatement(name):
    ts, counts, lists = STASH[name + "_ts"], STASH[name + "_counts"], STASH[name + "_lists"]
    docs, dlen = STASH[name + "_docs"].tobytes(), STASH[name + "_doc_len"]
    sent, slen = STASH[name + "_stash"].tobytes(), STASH[name + "_stash_len"]
    do, so = np.concatenate([[0], np.cumsum(dlen)]), np.concatenate([[0], np.cumsum(slen)])
    offs = np.concatenate([[0], np.cumsum(counts)])
    assert ts.size >= 40
    dj = DetectionJson(2000000, max_held=4096, device=0)
    assert dj.fetch_stash() == b"[]"
    st = Stash()
    for i in range(ts.size):
        t = _render(dj, lists[:, offs[i]:offs[i + 1]])
        if dlen[i] == 0:  # a NaN: no document, the history is unchanged
            with pytest.raises(capi.B200ddError) as e:
                dj.fetch(int(ts[i]))
            assert e.value.code == capi.ERR_NONFINITE
        else:
            doc = dj.fetch(int(ts[i]))
            assert doc == docs[do[i]:do[i + 1]]
            st.push(doc)
        got = dj.fetch_stash()
        assert got == sent[so[i]:so[i + 1]] == st.send(), i
        del t
    dj.close()


def test_ring_overflow_keeps_the_documents_and_loses_the_history():
    dj = DetectionJson(2000000, max_held=10, device=0)
    rng = np.random.default_rng(1)
    for i, n in enumerate((4, 4, 3, 2)):
        lists = [rng.uniform(1, 50, n) for _ in range(3)]
        t = _render(dj, lists)
        rc, doc = _fetch(dj, 1000 + i)
        assert doc == DetectionJson.render_host(*lists, 1000 + i, 2000000)
        assert rc == (capi.ERR_CAPACITY if i == 2 else capi.OK)
        if i < 2:
            assert dj.fetch_stash().startswith(b'{"timestamp":[1000,')
        else:
            with pytest.raises(capi.B200ddError) as e:
                dj.fetch_stash()
            assert e.value.code == capi.ERR_CAPACITY
        del t
    dj.close()


def test_list_overflow_and_misuse():
    dj = DetectionJson(2000000, max_held=1 << 19, device=0)
    with pytest.raises(capi.B200ddError) as e:  # nothing rendered
        dj.fetch(1)
    assert e.value.code == capi.ERR_ARG
    lists = large_lists("bounded_full")
    t = _render(dj, lists, count=N_FULL + 1)
    rc, doc = _fetch(dj, 1)
    assert rc == capi.ERR_CAPACITY and doc == b""
    assert dj.fetch_stash() == b"[]"  # nothing committed
    with pytest.raises(capi.B200ddError) as e:  # the render was consumed
        dj.fetch(1)
    assert e.value.code == capi.ERR_ARG
    t = _render(dj, lists)  # the full list itself renders whole
    rc, doc = _fetch(dj, 2)
    assert rc == capi.OK and doc == DetectionJson.render_host(*lists, 2, 2000000)
    out = np.empty(16, dtype=np.uint8)
    n = C.c_size_t()
    t = _render(dj, [a[:3] for a in lists])
    rc = capi.load().b200dd_detjson_fetch(dj._h, 3, capi.ptr(out), out.size, C.byref(n), None)
    assert rc == capi.ERR_CAPACITY and n.value > 16
    assert dj.fetch(3).startswith(b'{"timestamp":3,"delay":[')  # a too-small buffer leaves the render to fetch again
    del t
    dj.close()


# ---- the pipeline stage, on every submit path

FS, N = 200000, 40000
DET = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
N_CPI = 24
ZERO_REF = 9  # the CPI whose reference channel is zero: its solve fails


def _pipeline(**kw):
    return Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, clutter=(-5, 30), detection=DET, device=0,
                    map_json=True, **kw)


def _scenes():
    rng = np.random.default_rng(4)
    out = []
    for i in range(N_CPI):
        tg = [Target(int(rng.integers(8, 55)), float(rng.uniform(-400, 400)), float(rng.uniform(-35, -20)))
              for _ in range(int(rng.integers(1, 5)))]
        sc = make_scene(N, FS, seed=300 + i, targets=tg)
        out.append((np.zeros_like(sc.x) if i == ZERO_REF else sc.x, sc.y))
    return out


def _ts(i):  # 100 ms steps with two jumps past 300 s: the prune fires
    return 1731000000000 + 100 * i + 300050 * (i >= 14) + 300050 * (i >= 19)


@pytest.mark.parametrize("path", ["process_host", "submit_host", "submit_host_rspduo", "device_eager", "device_graph"])
def test_pipeline_stage_on_every_submit_path(path):
    import torch
    pipe = _pipeline(detection_json=True, max_held_detections=4096)
    assert pipe.fetch_detection_stash() == b"[]"
    g = pipe.geometry
    dx = torch.empty(N, dtype=torch.complex64, device="cuda")
    dy = torch.empty_like(dx)
    dmap = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    st = Stash()
    n_det = 0
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
        ts = _ts(i)
        if i == ZERO_REF:
            assert r["skipped"]
            with pytest.raises(capi.B200ddError) as e:
                pipe.fetch_detection_json(ts)
            assert e.value.code == capi.FILTER_FAILED
            assert pipe.fetch_detection_stash() == st.send()
            continue
        pipe.fetch_map_json(ts)
        d = r["detections"]
        doc = pipe.fetch_detection_json(ts)
        assert doc == DetectionJson.render_host(d.delay, d.doppler, d.snr, ts, FS), i
        if refdetjson.available():
            assert doc == refdetjson.detection_json(d.delay, d.doppler, d.snr, ts, FS)
        st.push(doc)
        assert pipe.fetch_detection_stash() == st.send(), i
        n_det += d.get_nDetections()
    assert n_det >= N_CPI
    pipe.close()


def test_pipeline_stage_needs_detection():
    with pytest.raises(capi.B200ddError) as e:
        Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, device=0, detection_json=True)
    assert e.value.code == capi.ERR_ARG


def test_pipeline_stage_changes_no_other_output():
    a = _pipeline(detection_json=True)
    b = _pipeline()
    for i, (x, y) in enumerate(_scenes()[:4]):
        ra, rb = a.process(x, y), b.process(x, y)
        assert np.array_equal(ra["map"], rb["map"])
        assert ra["noisePower"] == rb["noisePower"] and ra["maxPower"] == rb["maxPower"]
        da, db = ra["detections"], rb["detections"]
        assert np.array_equal(da.delay, db.delay) and np.array_equal(da.doppler, db.doppler)
        assert np.array_equal(da.snr, db.snr)
        assert a.fetch_map_json(i) == b.fetch_map_json(i)
