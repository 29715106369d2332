"""GPU: the pipeline's timing stage.  Every document is Timing::to_json's bytes of the names and times behind it (the
stand-alone render, which tests/golden pins to the reference) on every submit path; its keys are blah2's, in blah2's
order, for all 12 stage combinations blah2 can run; its times are device stage times that add up to the CPI time and
fit inside the host's wall time; /stash/timing is the restatement of api/stash/timing.js of the documents produced,
alone and in share sets; and with the stage on every other output is bit-identical to the stage off."""
import ctypes as C
import itertools
import json
import time

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import Pipeline, timing_render_host
from blah2_b200.scene import Target, make_scene
from oracle.stash_timing import Stash
from cpi_products import cpi_products
from test_shared_history_gpu import BAD, DET, DET_DIRECT, FS, METRICS, N, N_CPI, PATHS, TRK, Feeder, _scenes, _ts

pytestmark = pytest.mark.gpu

T_START = 1730999990000
CHAIN = ["extract_buffer", "spectrum", "clutter_filter", "ambiguity_processing", "detector", "output_radar_data"]


def _code(f):
    try:
        f()
        return capi.OK
    except capi.B200ddError as e:
        return e.code


def _expected_keys(spectrum, clutter, detection, tracker):
    return (["timestamp", "nCpi", "uptime_s", "uptime_days", "extract_buffer"] + (["spectrum"] if spectrum else [])
            + (["clutter_filter"] if clutter else []) + ["ambiguity_processing"] + (["detector"] if detection else [])
            + (["tracker"] if tracker else []) + ["output_radar_data", "cpi"])


def _check_document(pipe, doc, ts, n_cpi):
    """doc is Timing::to_json of the pipeline's names and times; returns the parsed document and those."""
    names, values = pipe.timing_values()
    assert doc == timing_render_host(T_START, ts, n_cpi, names, values)
    d = json.loads(doc)
    assert d["nCpi"] == n_cpi and d["timestamp"] == ts
    assert np.all(np.isfinite(values)) and np.all(values >= 0.0)
    return d, dict(zip(names, values))


COMBOS = list(itertools.product((False, True), (False, True), ("none", "detection", "tracker")))


@pytest.mark.parametrize("path", PATHS)
def test_documents_keys_and_times_for_every_stage_combination(path):
    for spectrum, clutter, det in COMBOS:
        kw = dict(roundHamming=True, device=0, spectrum_bandwidth=2000 if spectrum else None,
                  clutter=(-5, 30) if clutter else None, detection=DET if det != "none" else None)
        if det == "tracker":
            kw.update(tracker=TRK, max_tracks=1 << 12, max_track_history=32)
        pipe = Pipeline(-5, 60, -500, 500, FS, N, **kw)
        pipe.enable_timing_json(T_START)
        feed = Feeder(path, _scenes("filtered"))
        for k in range(3):
            t0 = time.perf_counter()
            feed.submit(pipe, k)  # device paths: the wall time also holds the feeder's copies
            pipe.fetch()
            if det == "tracker":
                pipe.fetch_track_json(_ts(k))
            wall = (time.perf_counter() - t0) * 1e3
            doc = pipe.fetch_timing_json(_ts(k))
            d, v = _check_document(pipe, doc, _ts(k), k + 1)
            assert list(d) == _expected_keys(spectrum, clutter, det != "none", det == "tracker"), (path, list(d))
            stages = [s for s in v if s != "cpi"]
            assert v["cpi"] >= sum(v[s] for s in stages) - 0.01 * len(stages)
            assert v["cpi"] <= wall, (v["cpi"], wall)
            assert (v["extract_buffer"] == 0.0) == path.startswith("device")
            assert v["ambiguity_processing"] > 0.0 and v["cpi"] > 0.0
        pipe.close()


def test_stage_off_and_on_give_identical_outputs_on_every_path():
    """Every product of the shared-history sequence (map, spectrum, max-hold, detection, IQ-data, track documents and
    stashes, fetch's results), with the timing stage on against off."""
    for config in ("filtered", "direct"):
        for path in PATHS:
            runs = []
            for on in (False, True):
                kw = dict(roundHamming=True, device=0, spectrum_bandwidth=2000, map_json=True, maxhold=True,
                          detection_json=True, max_held_detections=1 << 16, tracker=TRK, max_tracks=1 << 12,
                          max_track_history=32)
                if config == "filtered":
                    pipe = Pipeline(-5, 60, -500, 500, FS, N, clutter=(-5, 30), detection=DET, **kw)
                else:
                    pipe = Pipeline(-5, 60, -500, 500, FS, N, detection=DET_DIRECT, **kw)
                pipe.enable_iqdata_json(*METRICS)
                if on:
                    pipe.enable_timing_json(T_START)
                feed = Feeder(path, _scenes(config))
                out = []
                for k in range(14):
                    feed.submit(pipe, k)
                    out.append(cpi_products(pipe, _ts(k)))
                    if on:
                        code = _code(lambda: pipe.fetch_timing_json(_ts(k)))
                        assert code == (capi.FILTER_FAILED if (config, k) == ("filtered", BAD) else capi.OK)
                runs.append(out)
                pipe.close()
            assert runs[0] == runs[1], (config, path)


def _timing_pipeline(config):
    kw = dict(roundHamming=True, device=0, spectrum_bandwidth=2000, tracker=TRK, max_tracks=1 << 12,
              max_track_history=32)
    if config == "filtered":
        p = Pipeline(-5, 60, -500, 500, FS, N, clutter=(-5, 30), detection=DET, **kw)
    else:
        p = Pipeline(-5, 60, -500, 500, FS, N, detection=DET_DIRECT, **kw)
    p.enable_timing_json(T_START)
    return p


def _timing_products(pipe, k):
    """fetch(), the track fetch and the timing fetch of CPI k: (timing code, document, stash)."""
    pipe.fetch()
    _code(lambda: pipe.fetch_track_json(_ts(k)))
    code = _code(lambda: pipe.fetch_timing_json(_ts(k)))
    return code, (pipe.last_timing_doc if code == capi.OK else None), pipe.fetch_timing_stash()


@pytest.mark.parametrize("path", PATHS)
def test_stash_is_the_restatement_of_the_documents_produced(path):
    pipe = _timing_pipeline("filtered")
    assert pipe.fetch_timing_stash() == b"{}"
    feed = Feeder(path, _scenes("filtered"))
    st = Stash()
    n_docs = 0
    for k in range(N_CPI):
        feed.submit(pipe, k)
        code, doc, stash = _timing_products(pipe, k)
        if k == BAD:  # the failed solve: no document, no nCpi step, the stash unchanged
            assert code == capi.FILTER_FAILED
            assert _code(lambda: pipe.fetch_timing_json(_ts(k))) == capi.FILTER_FAILED
        else:
            assert code == capi.OK
            n_docs += 1
            _check_document(pipe, doc, _ts(k), n_docs)
            st.push(doc)
            assert _code(lambda: pipe.fetch_timing_json(_ts(k))) == capi.ERR_ARG  # once per CPI
        assert stash == st.send(), k
    assert len(st.output["cpi"]) == 20 and n_docs == N_CPI - 1
    pipe.close()


def test_values_the_history_cannot_hold_are_written_but_not_committed():
    pipe = _timing_pipeline("direct")
    feed = Feeder("submit_host", _scenes("direct"))
    st = Stash()
    lib = capi.load()
    out = np.empty(pipe.timing_json_max_bytes, dtype=np.uint8)
    n = C.c_size_t()
    for k in range(3):
        feed.submit(pipe, k)
        pipe.fetch()
        # with the tracker enabled the document waits for the track fetch
        assert lib.b200dd_pipeline_fetch_timing_json(pipe._h, _ts(k), capi.ptr(out), out.size, C.byref(n)) == capi.ERR_ARG
        pipe.fetch_track_json(_ts(k))
        before = pipe.fetch_timing_stash()
        for bad in (T_START - 1, 10 ** 15 + 1, 2 ** 64 - 1):  # wrapped uptime, timestamps of 16 and more digits
            rc = lib.b200dd_pipeline_fetch_timing_json(pipe._h, bad, capi.ptr(out), out.size, C.byref(n))
            assert rc == capi.ERR_ARG and n.value > 0
            assert json.loads(out[:n.value].tobytes())["nCpi"] == k + 1
            assert pipe.fetch_timing_stash() == before
        rc = lib.b200dd_pipeline_fetch_timing_json(pipe._h, _ts(k), capi.ptr(out), 8, C.byref(n))
        assert rc == capi.ERR_CAPACITY and n.value > 8
        doc = pipe.fetch_timing_json(_ts(k))
        assert json.loads(doc)["nCpi"] == k + 1
        st.push(doc)
        assert pipe.fetch_timing_stash() == st.send()
    assert b'"timestamp":[' in pipe.fetch_timing_stash()
    pipe.close()


def test_a_cfar_overflow_does_not_stop_the_document():
    """pfa 0.9 on a 606 x 801 map: about 4.4e5 CFAR detections against the list's 2^18 (as the tracker test)."""
    fs, n = 2000000, 800000
    det = dict(pfa=0.9, nGuard=2, nTrain=6, minDelay=-5, minDoppler=0.0, nCentroid=4)
    pipe = Pipeline(-5, 600, -1000, 1000, fs, n, roundHamming=True, detection=det, device=0, max_detections=16,
                    tracker=TRK)
    pipe.enable_timing_json(T_START)
    sc = make_scene(n, fs, seed=9, targets=[Target(40, 120.0, -20.0)])
    st = Stash()
    for i, y in enumerate([np.zeros_like(sc.y), sc.y, np.zeros_like(sc.y)]):
        pipe.submit_host(sc.x, y)
        pipe.fetch()
        code = _code(lambda: pipe.fetch_track_json(_ts(i)))
        assert code == (capi.ERR_CAPACITY if i == 1 else capi.OK)
        doc = pipe.fetch_timing_json(_ts(i))
        d, v = _check_document(pipe, doc, _ts(i), i + 1)
        assert "tracker" in d and (v["tracker"] == 0.0) == (i == 1)
        st.push(doc)
        assert pipe.fetch_timing_stash() == st.send()
    pipe.close()


def _alternate(pipes, path, config):
    P = len(pipes)
    feed = Feeder(path, _scenes(config))
    out = [None] * N_CPI
    for m, k in enumerate(range(N_CPI)):
        feed.submit(pipes[m % P], k)
        if m - P + 1 >= 0:
            j = m - P + 1
            out[j] = _timing_products(pipes[j % P], j)
    for j in range(max(N_CPI - P + 1, 0), N_CPI):
        out[j] = _timing_products(pipes[j % P], j)
    return out


def _shape(rec):
    """What a share set must reproduce: the code, the document without stage times, and the stash's keys and
    lengths."""
    code, doc, stash = rec
    d = json.loads(doc) if doc else None
    head = None if d is None else ([k for k in d], d["timestamp"], d["nCpi"], d["uptime_s"], d["uptime_days"])
    s = json.loads(stash)
    return code, head, [(k, len(v)) for k, v in s.items()], s.get("timestamp"), s.get("uptime_s")


@pytest.mark.parametrize("path", ["submit_host", "device_graph"])
@pytest.mark.parametrize("config", ["filtered", "direct"])
def test_share_sets_keep_one_timing_history(config, path):
    ref = _alternate([_timing_pipeline(config)], path, config)
    for P in (1, 2, 3, 6):
        pipes = [_timing_pipeline(config) for _ in range(P)]
        Pipeline.share_history(pipes)
        out = _alternate(pipes, path, config)
        st = Stash()
        for i, (g, r) in enumerate(zip(out, ref)):
            assert _shape(g) == _shape(r), (P, i)
            if g[1]:
                st.push(g[1])
            assert g[2] == st.send(), (P, i)
        for p in pipes:
            p.close()


def test_share_set_misuse_is_refused_and_commits_nothing():
    lib = capi.load()
    a, b = _timing_pipeline("filtered"), _timing_pipeline("filtered")
    other = _timing_pipeline("filtered")
    other.enable_timing_json(T_START + 1)
    arr = (C.c_void_p * 2)(a._h, other._h)
    assert lib.b200dd_pipeline_share_history(arr, 2) == capi.ERR_ARG  # different tStart
    plain = Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, device=0, spectrum_bandwidth=2000,
                     clutter=(-5, 30), detection=DET, tracker=TRK, max_tracks=1 << 12, max_track_history=32)
    arr = (C.c_void_p * 2)(a._h, plain._h)
    assert lib.b200dd_pipeline_share_history(arr, 2) == capi.ERR_ARG  # stage on one, off the other
    Pipeline.share_history([a, b])
    assert lib.b200dd_pipeline_enable_timing_json(a._h, T_START, None, None) == capi.ERR_ARG
    feed = Feeder("submit_host", _scenes("filtered"))
    feed.submit(a, 0)
    feed.submit(b, 1)
    assert _code(lambda: a.fetch_timing_json(_ts(0))) == capi.ERR_ARG  # before its fetch
    a.fetch()
    a.fetch_track_json(_ts(0))
    b.fetch()
    b.fetch_track_json(_ts(1))
    b.fetch_timing_json(_ts(1))
    stash = b.fetch_timing_stash()
    assert _code(lambda: a.fetch_timing_json(_ts(0))) == capi.ERR_ARG  # older than the set's last commit
    assert a.fetch_timing_stash() == stash and json.loads(stash)["timestamp"] == [_ts(1)]
    for p in (a, b, other, plain):
        p.close()
