"""GPU: the device tracker is blah2's Tracker + Track::to_json, byte for byte: the stand-alone handle against every
document of tests/golden/track_docs.npz through process_host and process_device, against the CPU model and the
compiled reference on random sequences, its capacity limits and reset; the pipeline stage against the model (and the
compiled reference, where built) fed with the pipeline's own detection lists on every submit path."""
import ctypes as C
import json

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import Pipeline, Tracker
from blah2_b200.scene import Target, make_scene
from oracle import reftracker
from oracle.track_model import TrackModel
from track_sequences import load, matches, random_large_sequence, random_sequence, stored

pytestmark = pytest.mark.gpu
Z = load()
NAMES = [str(n) for n in Z["names"]]


def _dev(d, f, s):
    import torch
    t = [torch.from_numpy(np.ascontiguousarray(a if len(a) else [0.0], dtype=np.float64)).cuda() for a in (d, f, s)]
    return t + [torch.tensor([len(d)], dtype=torch.int32, device="cuda")]


def _process(tr, path, d, f, s, ts):
    if path == "host":
        tr.process_host(d, f, s, ts)
        return None
    t = _dev(d, f, s)
    tr.process_device(*t, ts)
    return t  # alive until the fetch


def _fetch(tr, ts):
    try:
        return capi.OK, tr.fetch(ts)
    except capi.B200ddError as e:
        return e.code, b""


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("name", NAMES)
def test_stored_sequences(name, path):
    params, (max_tracks, max_hist), cpis, docs = stored(Z, name)
    tr = Tracker(*params, max_tracks=max_tracks, max_history=max_hist, device=0)  # the exact limits fit
    for i, ((d, f, s, ts), want) in enumerate(zip(cpis, docs)):
        keep = _process(tr, path, d, f, s, ts)
        rc, doc = _fetch(tr, ts)
        del keep
        if want[3]:
            assert rc == capi.ERR_NONFINITE and doc == b"", (name, i)
        else:
            assert rc == capi.OK and matches(doc, want), (name, i, doc[:200])
    tr.close()


def test_random_sequences_match_model_and_reference():
    rng = np.random.default_rng(77)
    n_docs = 0
    for k in range(150):
        params, cpis = random_sequence(rng)
        tr = Tracker(*params, max_tracks=4096, max_history=128, device=0)
        mod = TrackModel(*params)
        ref = reftracker.RefTracker(*params) if reftracker.available() else None
        for d, f, s, ts in cpis:
            keep = _process(tr, "device" if k % 2 else "host", d, f, s, ts)
            mod.process(d, f, ts)
            want = mod.to_json(ts, capi.format_track_doubles)
            rc, doc = _fetch(tr, ts)
            del keep
            if want is None:
                assert rc == capi.ERR_NONFINITE
            else:
                assert rc == capi.OK and doc == want
            if ref is not None:
                r = ref.process(d, f, s, ts)
                assert want is None or r == want
            n_docs += 1
        tr.close()
    assert n_docs > 1500


def test_random_sequences_with_thousands_of_tracks():
    """Thousands of tracks at entry, removals on both sides of the update kernel's 1024-track chunks."""
    rng = np.random.default_rng(8192)
    most = 0
    for k in range(3):
        params, cpis = random_large_sequence(rng)
        tr = Tracker(*params, max_tracks=1 << 16, max_history=64, device=0)
        mod = TrackModel(*params)
        ref = reftracker.RefTracker(*params) if reftracker.available() else None
        for d, f, s, ts in cpis:
            most = max(most, len(mod.tracks))
            keep = _process(tr, "device" if k % 2 else "host", d, f, s, ts)
            mod.process(d, f, ts)
            want = mod.to_json(ts, capi.format_track_doubles)
            assert tr.fetch(ts) == want
            del keep
            if ref is not None:
                assert ref.process(d, f, s, ts) == want
        tr.close()
    assert most > 4096


def test_fetch_repeats_and_small_buffer():
    params, lim, cpis, docs = stored(Z, "assoc")
    tr = Tracker(*params, max_tracks=lim[0], max_history=lim[1], device=0)
    for d, f, s, ts in cpis[:10]:
        tr.process_host(d, f, s, ts)
    a = tr.fetch(5)
    assert tr.fetch(5) == a and len(a) > 200  # fetching renders, it does not advance
    out = np.empty(16, dtype=np.uint8)
    n = C.c_size_t()
    rc = capi.load().b200dd_tracker_fetch(tr._h, 5, capi.ptr(out), out.size, C.byref(n), None)
    assert rc == capi.ERR_CAPACITY and n.value == len(a)
    tr.close()


@pytest.mark.parametrize("which", ["tracks", "history"])
def test_overflow_and_reset(which):
    name = "assoc"
    params, (max_tracks, max_hist), cpis, docs = stored(Z, name)
    if which == "tracks":
        max_tracks -= 1
    else:
        max_hist -= 1
    tr = Tracker(*params, max_tracks=max_tracks, max_history=max_hist, device=0)
    mod = TrackModel(*params)
    first = None  # the first CPI after which the model holds more tracks, or a longer history, than the limits
    for i, (d, f, s, ts) in enumerate(cpis):
        mod.process(d, f, ts)
        longest = max((len(t["hist"]) for t in mod.tracks), default=0)
        if first is None and (len(mod.tracks) > max_tracks or longest > max_hist):
            first = i
    over = None
    for i, ((d, f, s, ts), want) in enumerate(zip(cpis, docs)):
        tr.process_host(d, f, s, ts)
        rc, doc = _fetch(tr, ts)
        if rc == capi.ERR_CAPACITY:
            over = i if over is None else over
            assert doc == b""
            n = C.c_size_t(123)
            out = np.empty(1 << 20, dtype=np.uint8)
            assert capi.load().b200dd_tracker_fetch(tr._h, ts, capi.ptr(out), out.size, C.byref(n), None) == \
                capi.ERR_CAPACITY and n.value == 0
        else:
            assert over is None and rc == capi.OK and matches(doc, want), i  # overflowed stays overflowed
    assert over is not None and over == first
    tr.reset()
    for i, ((d, f, s, ts), want) in enumerate(zip(cpis[:over], docs[:over])):  # as new
        tr.process_host(d, f, s, ts)
        assert matches(tr.fetch(ts), want), i
    tr.close()


# ---- the pipeline stage, on every submit path

FS, N = 200000, 40000
DET = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
# no clutter filter, and CFAR over delay 0 and Doppler 0: the direct path is detected near (0.4 bins, 0 Hz), inside the
# association window (|Doppler| < 1 / cpi = 5 Hz), so every CPI associates and tracks coast into the documents
DET_DIRECT = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=-5, minDoppler=0.0, nCentroid=4)
TRK = dict(M=2, N=3, delete=4, maxAcc=30, fc=204640000)
N_CPI = 16
ZERO_REF = 6  # the CPI whose reference channel is zero: its solve fails


def _pipeline(direct=False, **kw):
    if direct:
        return Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, detection=DET_DIRECT, device=0, **kw)
    return Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, clutter=(-5, 30), detection=DET, device=0, **kw)


def _scenes(zero_ref=True):
    rng = np.random.default_rng(5)
    out = []
    for i in range(N_CPI):
        tg = [Target(int(rng.integers(8, 55)), float(rng.uniform(-400, 400)), float(rng.uniform(-35, -20)))
              for _ in range(int(rng.integers(1, 5)))]
        sc = make_scene(N, FS, seed=500 + i, targets=tg)
        out.append((np.zeros_like(sc.x) if zero_ref and i == ZERO_REF else sc.x, sc.y))
    return out


def _params(pipe):
    return (TRK["M"], TRK["N"], TRK["delete"], pipe.geometry.cpi, float(TRK["maxAcc"]), FS, TRK["fc"])


@pytest.mark.parametrize("mode", ["filtered", "direct"])
@pytest.mark.parametrize("path", ["process_host", "submit_host", "submit_host_rspduo", "device_eager", "device_graph"])
def test_pipeline_stage_on_every_submit_path(path, mode):
    """filtered: the clutter filter removes the direct path, nothing associates and one CPI's solve fails; direct:
    the direct path associates every CPI, so the documents carry the delays and Doppler values the pipeline's device
    list handed the tracker."""
    import torch
    direct = mode == "direct"
    pipe = _pipeline(direct, tracker=TRK, max_tracks=1 << 14, max_track_history=64)
    mod = TrackModel(*_params(pipe))
    ref = reftracker.RefTracker(*_params(pipe)) if reftracker.available() else None
    g = pipe.geometry
    dx = torch.empty(N, dtype=torch.complex64, device="cuda")
    dy = torch.empty_like(dx)
    dmap = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    n_det = n_sent = 0
    for i, (x, y) in enumerate(_scenes(zero_ref=not direct)):
        if path == "process_host":
            r = pipe.process(x, y)
        else:
            if path == "submit_host":
                pipe.submit_host(x, y)
            elif path == "submit_host_rspduo":
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
        ts = 1731000000000 + 200 * i
        if i == ZERO_REF and not direct:
            assert r["skipped"]
            for _ in range(2):
                with pytest.raises(capi.B200ddError) as e:
                    pipe.fetch_track_json(ts)
                assert e.value.code == capi.FILTER_FAILED
            continue
        d = r["detections"]
        doc = pipe.fetch_track_json(ts)
        assert pipe.fetch_track_json(ts) == doc  # later calls for the same CPI render again, the tracker is run once
        mod.process(d.delay, d.doppler, ts)
        assert doc == mod.to_json(ts, capi.format_track_doubles), i
        if ref is not None:
            assert doc == ref.process(d.delay, d.doppler, d.snr, ts)
        n_det += d.get_nDetections()
        n_sent += json.loads(doc)["nCoasting"]
    assert n_det >= N_CPI
    assert (n_sent > N_CPI) == direct  # only the direct path's associations put tracks into the documents
    pipe.close()


def test_pipeline_stage_needs_detection():
    with pytest.raises(capi.B200ddError) as e:
        Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, device=0, tracker=TRK)
    assert e.value.code == capi.ERR_ARG


@pytest.mark.parametrize("path", ["process_host", "device_graph"])
def test_pipeline_stage_changes_no_other_output(path):
    """Every other output of a pipeline with the tracker equals that of one without it, bit for bit, over CPIs that
    include a failed solve, on the host path and on graph-replayed device submits."""
    import torch
    a = _pipeline(tracker=TRK, map_json=True, detection_json=True, maxhold=True)
    b = _pipeline(map_json=True, detection_json=True, maxhold=True)
    g = a.geometry
    dx = torch.empty(N, dtype=torch.complex64, device="cuda")
    dy = torch.empty_like(dx)
    maps = [torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda") for _ in range(2)]

    def code(fn, *args):
        try:
            return fn(*args)
        except capi.B200ddError as e:
            return e.code

    for i, (x, y) in enumerate(_scenes()[:ZERO_REF + 2]):
        if path == "process_host":
            ra, rb = a.process(x, y), b.process(x, y)
            ma, mb = ra["map"], rb["map"]
        else:
            dx.copy_(torch.from_numpy(x.astype(np.complex64)))
            dy.copy_(torch.from_numpy(y.astype(np.complex64)))
            torch.cuda.synchronize()
            for p, m in zip((a, b), maps):
                (p.prepare_device if i == 0 else p.submit_device)(dx, dy, m)
            ra, rb = a.fetch(), b.fetch()
            ma, mb = (m.cpu().numpy() for m in maps)
        assert ra["skipped"] == rb["skipped"] == (i == ZERO_REF)
        code(a.fetch_track_json, i)
        if not ra["skipped"]:
            assert np.array_equal(ma, mb)
        assert ra["noisePower"] == rb["noisePower"] and ra["maxPower"] == rb["maxPower"]
        da, db = ra["detections"], rb["detections"]
        assert np.array_equal(da.delay, db.delay) and np.array_equal(da.doppler, db.doppler)
        assert np.array_equal(da.snr, db.snr)
        assert code(a.fetch_map_json, i) == code(b.fetch_map_json, i)
        assert code(a.fetch_maxhold, i) == code(b.fetch_maxhold, i)
        assert code(a.fetch_detection_json, i) == code(b.fetch_detection_json, i)
        assert a.fetch_detection_stash() == b.fetch_detection_stash()


def test_pipeline_cfar_overflow_leaves_the_tracker_unchanged():
    """A CPI whose CFAR list overflows (pfa 0.9 on a 606 x 801 map: about 4.4e5 CFAR detections against the list's
    2^18) returns ERR_CAPACITY with nothing written, on every call, and the tracker does not run: the next CPI's
    document is the model's with that CPI left out.  The CPIs around it have an all-zero surveillance channel, whose
    map is exactly zero and has no detections.  Had the tracker taken the truncated list (2^18 detections x 9
    hypotheses), the next fetch would report an overflowed tracker instead."""
    fs, n = 2000000, 800000
    det = dict(pfa=0.9, nGuard=2, nTrain=6, minDelay=-5, minDoppler=0.0, nCentroid=4)
    pipe = Pipeline(-5, 600, -1000, 1000, fs, n, roundHamming=True, detection=det, device=0, max_detections=16,
                    tracker=TRK)
    mod = TrackModel(TRK["M"], TRK["N"], TRK["delete"], pipe.geometry.cpi, float(TRK["maxAcc"]), fs, TRK["fc"])
    sc = make_scene(n, fs, seed=9, targets=[Target(40, 120.0, -20.0)])
    quiet = np.zeros_like(sc.y)
    lib = capi.load()
    out = np.empty(1 << 16, dtype=np.uint8)
    for i, y in enumerate([quiet, sc.y, quiet]):
        r = pipe.process(sc.x, y, want_map=False)
        ts = 1731000000000 + 400 * i
        if i == 1:
            for _ in range(2):
                nb = C.c_size_t(123)
                rc = lib.b200dd_pipeline_fetch_track_json(pipe._h, ts, capi.ptr(out), out.size, C.byref(nb))
                assert rc == capi.ERR_CAPACITY and nb.value == 0
            continue
        assert r["detections"].get_nDetections() == 0
        mod.process([], [], ts)
        assert pipe.fetch_track_json(ts) == mod.to_json(ts, capi.format_track_doubles)
    pipe.close()
