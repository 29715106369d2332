"""GPU: a share set of pipelines used alternately keeps one max-hold window, one detection history, one IQ-data history
and one tracker.  After every fetch, with P members taking CPIs round-robin, every stash and track document -- and
every per-CPI product -- equals that of one unshared pipeline given the same CPIs one after another, on every submit
path; the same alternation without sharing does not; misuse is refused without consuming or committing anything."""
import ctypes as C

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import Pipeline
from blah2_b200.scene import Target, make_scene
from cpi_products import cpi_products

pytestmark = pytest.mark.gpu

FS, N = 200000, 40000
DET = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
DET_DIRECT = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=-5, minDoppler=0.0, nCentroid=4)
TRK = dict(M=2, N=3, delete=4, maxAcc=30, fc=204640000)
METRICS = (0.0, -1.005, 1e21)
N_CPI = 26
BAD = 12   # filtered: a zero reference channel, its solve fails; direct: an all-zero CPI the max-hold rejects
GAP = 17   # from this CPI on the timestamps jump by 301 s: detection.js prunes everything before
PATHS = ["submit_host", "submit_host_rspduo", "device_eager", "device_graph"]


def _pipeline(config):
    kw = dict(roundHamming=True, device=0, spectrum_bandwidth=2000, map_json=True, maxhold=True, detection_json=True,
              max_held_detections=1 << 16, tracker=TRK, max_tracks=1 << 12, max_track_history=32)
    if config == "filtered":
        p = Pipeline(-5, 60, -500, 500, FS, N, clutter=(-5, 30), detection=DET, **kw)
    else:
        p = Pipeline(-5, 60, -500, 500, FS, N, detection=DET_DIRECT, **kw)
    p.enable_iqdata_json(*METRICS)
    return p


_SCENES = {}


def _scenes(config):
    if config not in _SCENES:
        rng = np.random.default_rng(11)
        out = []
        for i in range(N_CPI):
            tg = [Target(int(rng.integers(8, 55)), float(rng.uniform(-400, 400)), float(rng.uniform(-35, -20)))
                  for _ in range(int(rng.integers(1, 4)))]
            sc = make_scene(N, FS, seed=700 + i, targets=tg)
            x, y = sc.x, sc.y
            if i == BAD:
                x = np.zeros_like(x)
                if config == "direct":
                    y = np.zeros_like(y)
            out.append((x, y))
        _SCENES[config] = out
    return _SCENES[config]


def _ts(i):
    return 1731000000000 + 100 * i + (301000 if i >= GAP else 0)


class Feeder:
    """Submits CPI k of a scene list to a pipeline on one path; device paths use per-pipeline buffers, and the graph
    path prepares each pipeline's buffers with its first CPI."""

    def __init__(self, path, scenes):
        import torch
        self.torch = torch
        self.path, self.scenes = path, scenes
        self.bufs, self.keep = {}, {}

    def submit(self, pipe, k):
        x, y = self.scenes[k]
        if self.path == "submit_host":
            self.keep[id(pipe)] = (x, y)
            pipe.submit_host(x, y)
        elif self.path == "submit_host_rspduo":
            iq = np.empty((N, 4), dtype="<i2")
            iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = x.real, x.imag, y.real, y.imag
            self.keep[id(pipe)] = iq
            pipe.submit_host_rspduo(iq)
        else:
            torch = self.torch
            first = id(pipe) not in self.bufs
            if first:
                g = pipe.geometry
                dx = torch.empty(N, dtype=torch.complex64, device="cuda")
                self.bufs[id(pipe)] = (dx, torch.empty_like(dx),
                                       torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64,
                                                   device="cuda"))
            dx, dy, dm = self.bufs[id(pipe)]
            dx.copy_(torch.from_numpy(x.astype(np.complex64)))
            dy.copy_(torch.from_numpy(y.astype(np.complex64)))
            torch.cuda.synchronize()
            if self.path == "device_graph" and first:
                pipe.prepare_device(dx, dy, dm)
            else:
                pipe.submit_device(dx, dy, dm)


_REFS = {}


def _reference(config, path):
    """One unshared pipeline, every CPI submitted, fetched and its products fetched in turn (device paths eager)."""
    key = (config, "device" if path.startswith("device") else path)
    if key not in _REFS:
        pipe = _pipeline(config)
        feed = Feeder("device_eager" if key[1] == "device" else path, _scenes(config))
        out = []
        for k in range(N_CPI):
            feed.submit(pipe, k)
            out.append(cpi_products(pipe, _ts(k)))
        pipe.close()
        _REFS[key] = out
    return _REFS[key]


def _alternate(pipes, feed, ks, out, between=None):
    """CPIs ks on pipes round-robin: submit(k) on member k mod P, then fetch the CPI P - 1 before it."""
    P = len(pipes)
    for n, k in enumerate(ks):
        feed.submit(pipes[n % P], k)
        if between:
            between(n, k)
        if n - P + 1 >= 0:
            j = n - P + 1
            out[ks[j]] = cpi_products(pipes[j % P], _ts(ks[j]))
    for j in range(max(len(ks) - P + 1, 0), len(ks)):
        out[ks[j]] = cpi_products(pipes[j % P], _ts(ks[j]))


def _assert_same(got, ref):
    for i, (g, r) in enumerate(zip(got, ref)):
        for a, b in zip(g, r):
            assert a == b, f"CPI {i}: {a[0]} differs"


def test_sequence_exercises_every_case():
    for config in ("filtered", "direct"):
        ref = _reference(config, "submit_host")
        rec = dict((name, v) for name, v, *_ in ref[BAD])
        assert ref[BAD][0][1][0] == (config == "filtered")  # the failed solve skips the CPI
        assert rec["maxhold"] == (capi.FILTER_FAILED if config == "filtered" else capi.ERR_NONFINITE)
        held = [dict((n, v) for n, v, *_ in r)["iqdata_stash"].count(b",[]") + 1 for r in ref[1:]]
        assert max(held) == 20 and held[-1] == 20  # the IQ-data window fills and evicts
        stashes = [dict((n, v) for n, v, *_ in r)["detection_stash"] for r in ref]
        assert len(stashes[GAP]) < len(stashes[GAP - 1])  # the 300 s prune ran
        tracks = [dict((n, v) for n, v, *_ in r)["track"] for r in ref]
        assert len({t for t in tracks if isinstance(t, bytes)}) > N_CPI // 2


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("config", ["filtered", "direct"])
def test_shared_alternation_equals_one_pipeline(config, path):
    ref = _reference(config, path)
    for P in (1, 2, 3, 6):
        pipes = [_pipeline(config) for _ in range(P)]
        Pipeline.share_history(pipes)
        out = [None] * N_CPI
        _alternate(pipes, Feeder(path, _scenes(config)), list(range(N_CPI)), out)
        _assert_same(out, ref)
        for p in pipes:
            p.close()


def test_unshared_alternation_differs():
    ref = _reference("filtered", "submit_host")
    pipes = [_pipeline("filtered") for _ in range(3)]
    out = [None] * N_CPI
    _alternate(pipes, Feeder("submit_host", _scenes("filtered")), list(range(N_CPI)), out)
    for p in pipes:
        p.close()
    differ = {name for g, r in zip(out, ref) for (name, a, *_), (_, b, *_) in zip(g, r) if a != b}
    assert {"maxhold", "detection_stash", "iqdata_stash"} <= differ
    assert not differ & {"fetch", "map", "spectrum", "detection", "iqdata"}  # the per-CPI products agree


def test_misuse_is_refused_and_changes_nothing():
    ref = _reference("filtered", "submit_host")
    pipes = [_pipeline("filtered") for _ in range(3)]
    lib = capi.load()

    def arr(ps):
        return (C.c_void_p * len(ps))(*[p._h for p in ps])

    other = _pipeline("filtered")
    bare = Pipeline(-5, 60, -500, 500, FS, N, clutter=(-5, 30), detection=DET, device=0, maxhold=True)
    assert lib.b200dd_pipeline_share_history(arr([other, other]), 2) == capi.ERR_ARG
    assert lib.b200dd_pipeline_share_history(arr([other, bare]), 2) == capi.ERR_ARG
    Pipeline.share_history(pipes)
    assert lib.b200dd_pipeline_share_history(arr([other, pipes[0]]), 2) == capi.ERR_ARG
    keep = _pipeline("filtered")
    Pipeline.share_history([other, keep])  # the refusals left other unshared
    feed = Feeder("submit_host", _scenes("filtered"))
    tp = capi.TrackerParams(2, 3, 4, 0.0, 30.0, 0, 204640000)
    n = C.c_size_t()

    def between(step, k):
        if step not in (4, 9):
            return
        with pytest.raises(capi.B200ddError) as e:  # CPI k is the newest of three unfetched
            pipes[step % 3].fetch()
        assert e.value.code == capi.ERR_ARG
        with pytest.raises(capi.B200ddError) as e:  # the member's CPI k is not fetched
            feed.submit(pipes[step % 3], k)
        assert e.value.code == capi.ERR_ARG
        with pytest.raises(capi.B200ddError) as e:  # the tracker takes a CPI only after its fetch
            pipes[step % 3].fetch_track_json(_ts(k))
        assert e.value.code == capi.ERR_ARG
        h = pipes[(step + 1) % 3]._h
        assert lib.b200dd_pipeline_enable_maxhold(h, C.byref(n)) == capi.ERR_ARG
        assert lib.b200dd_pipeline_enable_detection_json(h, 1 << 16, None, None) == capi.ERR_ARG
        assert lib.b200dd_pipeline_enable_tracker(h, C.byref(tp), 1 << 12, 32, None) == capi.ERR_ARG
        assert lib.b200dd_pipeline_enable_iqdata_json(h, *METRICS, None, None) == capi.ERR_ARG
        assert lib.b200dd_pipeline_enable_spectrum(h, 2000.0, None) == capi.ERR_ARG

    out = [None] * N_CPI
    _alternate(pipes, feed, list(range(N_CPI)), out, between)
    _assert_same(out, ref)
    # a product fetch for a CPI older than that product's last commit
    last = (N_CPI - 1) % 3
    for i, p in enumerate(pipes):
        if i == last:
            continue
        for f in (lambda: p.fetch_maxhold(1), lambda: p.fetch_track_json(1), lambda: p.fetch_detection_json(1),
                  lambda: p.fetch_iqdata_json(1)):
            with pytest.raises(capi.B200ddError) as e:
                f()
            assert e.value.code == capi.ERR_ARG
    assert pipes[last].fetch_detection_stash() == dict((n, v) for n, v, *_ in ref[-1])["detection_stash"]
    for p in pipes + [other, keep, bare]:
        p.close()


def test_destroying_a_member_keeps_the_others_working():
    ref = _reference("filtered", "submit_host")
    pipes = [_pipeline("filtered") for _ in range(3)]
    Pipeline.share_history(pipes)
    feed = Feeder("submit_host", _scenes("filtered"))
    out = [None] * N_CPI
    _alternate(pipes, feed, list(range(10)), out)
    pipes[1].close()
    _alternate([pipes[0], pipes[2]], feed, list(range(10, N_CPI)), out)
    _assert_same(out, ref)
    pipes[0].close()
    pipes[2].close()
