"""GPU: the max-hold document blah2's API serves at /stash/map, kept and rendered on the device, is the API's, byte
for byte: the device cell formatter against the host one, the stand-alone handle against tests/golden/maxhold_docs.npz
(the compiled reference's map documents through the stash restatement) after every CPI, and the pipeline stage
against the restatement applied to the pipeline's own map documents, on every submit path."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import MaxHold, Pipeline
from blah2_b200.scene import Target, make_scene
from map_json_maps import k_grid
from maxhold_maps import N_SEQ, SEQS, seq_map, timestamp, zero_cell
from oracle.stash_maxhold import Stash

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def test_device_cell_formatter_equals_host_formatter():
    z = gold("map_json_values")
    rng = np.random.default_rng(13)
    sets = [k_grid()[1].ravel(), z["small"], z["bits"].view(np.float64),
            rng.integers(0, 2 ** 64, 1 << 24, dtype=np.uint64).view(np.float64)]
    for vals in sets:
        host = capi.format_maxhold_doubles(vals)
        dev = capi.format_maxhold_doubles(vals, device=0)
        if host != dev:
            bad = [(vals[i], dev[i], host[i]) for i in range(vals.size) if dev[i] != host[i]]
            pytest.fail(f"{len(bad)} of {vals.size} differ: {bad[:5]}")


class Expected:
    """The fixture's /stash/map documents of one sequence, one per CPI (None: the CPI has no document)."""

    def __init__(self, name):
        z = gold("maxhold_docs")
        self.metrics = z[name + "_metrics"]
        self.lens = z[name + "_len"]
        self.sha = z[name + "_sha256"]
        self.docs = z[name + "_docs"].tobytes() if name + "_docs" in z else None
        self.offs = np.concatenate([[0], np.cumsum(self.lens)])

    def check(self, i, doc):
        assert self.lens[i] > 0
        if self.docs is not None:
            assert doc == self.docs[self.offs[i]:self.offs[i + 1]]
        assert len(doc) == self.lens[i]
        assert hashlib.sha256(doc).digest() == self.sha[i].tobytes()


def _run_sequence(name, dtype, bad_cell=None, bad_noise=None):
    """Pushes the sequence's CPIs into a new handle and checks the fetch after every one.  The "zero_cpi" CPI keeps
    its zero cell, or gets bad_cell there instead, or its clean map with noisePower bad_noise."""
    import torch
    spec = SEQS[name]
    exp = Expected(name)
    _, delay, doppler = seq_map(spec, 0)
    mh = MaxHold(delay, doppler, spec["fs"], device=0)
    for i in range(N_SEQ):
        m = seq_map(spec, i)[0]
        noise, maxp = (float(v) for v in exp.metrics[i])
        rejected = spec.get("zero_cpi") == i
        if rejected and bad_cell is not None:
            m[zero_cell(spec)] = bad_cell
        if rejected and bad_noise is not None:
            m, noise = seq_map(spec, i, with_zero=False)[0], bad_noise
        mh.push_device(torch.from_numpy(m).to("cuda", dtype), noise, maxp)
        if rejected:
            assert exp.lens[i] == 0
            with pytest.raises(capi.B200ddError) as e:
                mh.fetch(timestamp(spec, i))
            assert e.value.code == capi.ERR_NONFINITE
        else:
            exp.check(i, mh.fetch(timestamp(spec, i)))
    assert len(mh.fetch(0)) <= mh.max_bytes
    mh.close()


@pytest.mark.parametrize("dtype", ["complex64", "complex128"])
@pytest.mark.parametrize("name", list(SEQS))
def test_sequences_equal_the_fixture(name, dtype):
    import torch
    _run_sequence(name, getattr(torch, dtype))


@pytest.mark.parametrize("bad", ["nan_cell", "inf_cell", "nan_noise", "inf_noise"])
def test_rejected_cpis_leave_the_window_alone(bad):
    import torch
    kind, what = bad.split("_")
    v = float(kind)
    _run_sequence("medium", torch.complex64, bad_cell=v if what == "cell" else None,
                  bad_noise=v if what == "noise" else None)


def test_misuse():
    import torch
    spec = SEQS["small"]
    m, delay, doppler = seq_map(spec, 0)
    mh = MaxHold(delay, doppler, spec["fs"], device=0)
    with pytest.raises(capi.B200ddError) as e:  # nothing held yet
        mh.fetch(1)
    assert e.value.code == capi.ERR_ARG
    d = torch.from_numpy(m).cuda()
    for noise in (1.0000001e7, -2e7):
        with pytest.raises(capi.B200ddError) as e:
            mh.push_device(d, noise, 300.0)
        assert e.value.code == capi.ERR_ARG
    with pytest.raises(capi.B200ddError) as e:  # the rejected argument pushed nothing
        mh.fetch(1)
    assert e.value.code == capi.ERR_ARG
    mh.push_device(d, 1e7, 300.0)  # the bound itself is accepted
    assert mh.fetch(1).startswith(b'{"timestamp":1,"nRows":17,"nCols":33,"noisePower":10000000,"maxPower":300,')
    out = np.empty(16, dtype=np.uint8)
    n = C.c_size_t()
    rc = capi.load().b200dd_maxhold_fetch(mh._h, 1, capi.ptr(out), out.size, C.byref(n), None)
    assert rc == capi.ERR_CAPACITY and n.value > 16
    mh.close()


# ---- the pipeline stage against the restatement of the stash applied to the pipeline's own map documents

FS, N = 200000, 40000
DET = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
N_CPI = 26
ZERO_REF = 12  # the CPI whose reference channel is zero: its solve fails


def _pipeline(**kw):
    return Pipeline(-5, 60, -500, 500, FS, N, roundHamming=True, clutter=(-5, 30), detection=DET, device=0, **kw)


def _scenes():
    rng = np.random.default_rng(3)
    out = []
    for i in range(N_CPI):
        tg = [Target(int(rng.integers(8, 55)), float(rng.uniform(-400, 400)), float(rng.uniform(-35, -20)))
              for _ in range(int(rng.integers(1, 4)))]
        sc = make_scene(N, FS, seed=100 + i, targets=tg)
        x = np.zeros_like(sc.x) if i == ZERO_REF else sc.x
        out.append((x, sc.y))
    return out


def _after_cpi(pipe, stash, ts, i, docs):
    """Fetches CPI i's map document and max-hold document and checks the latter against the restatement."""
    r = pipe.fetch()
    if i == ZERO_REF:
        assert r["skipped"]
        for fetch in (pipe.fetch_map_json, pipe.fetch_maxhold):
            with pytest.raises(capi.B200ddError) as e:
                fetch(ts)
            assert e.value.code == capi.FILTER_FAILED
        docs.append(None)
        return
    assert not r["skipped"]
    stash.push(pipe.fetch_map_json(ts))
    doc = pipe.fetch_maxhold(ts)
    assert doc == stash.send(), f"CPI {i}"
    docs.append(doc)


def test_pipeline_stage_on_the_host_and_eager_paths():
    import torch
    scenes = _scenes()
    pipe = _pipeline(map_json=True, maxhold=True)
    assert pipe.maxhold_max_bytes > 0
    with pytest.raises(capi.B200ddError) as e:  # nothing submitted yet
        pipe.fetch_maxhold(1)
    assert e.value.code == capi.ERR_ARG
    g = pipe.geometry
    dx = torch.empty(N, dtype=torch.complex64, device="cuda")
    dy = torch.empty_like(dx)
    dmap = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    stash, docs = Stash(), []
    for i, (x, y) in enumerate(scenes):
        path = i % 3
        if path == 0:
            pipe.submit_host(x, y)
        elif path == 1:  # the scene's samples are integers
            iq = np.empty((N, 4), dtype="<i2")
            iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = x.real, x.imag, y.real, y.imag
            pipe.submit_host_rspduo(iq)
        else:
            dx.copy_(torch.from_numpy(x.astype(np.complex64)))
            dy.copy_(torch.from_numpy(y.astype(np.complex64)))
            torch.cuda.synchronize()
            pipe.submit_device(dx, dy, dmap)
        _after_cpi(pipe, stash, 1731000000000 + 100 * i, i, docs)
    assert len(stash.held) == 20
    plain = _pipeline()
    with pytest.raises(capi.B200ddError) as e:  # the stage is not enabled
        plain.fetch_maxhold(1)
    assert e.value.code == capi.ERR_ARG


def _device_run(graph):
    """All CPIs on the device path of a new pipeline: eager, or replayed from a graph prepared on fixed buffers
    whose contents are replaced before every CPI (prepare_device runs the chain once: it is CPI 0's submit)."""
    import torch
    pipe = _pipeline(map_json=True, maxhold=True)
    g = pipe.geometry
    dx = torch.empty(N, dtype=torch.complex64, device="cuda")
    dy = torch.empty_like(dx)
    dmap = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    stash, docs = Stash(), []
    for i, (x, y) in enumerate(_scenes()):
        dx.copy_(torch.from_numpy(x.astype(np.complex64)))
        dy.copy_(torch.from_numpy(y.astype(np.complex64)))
        torch.cuda.synchronize()
        if graph and i == 0:
            pipe.prepare_device(dx, dy, dmap)
        else:
            pipe.submit_device(dx, dy, dmap)
        _after_cpi(pipe, stash, 5 + i, i, docs)
    pipe.close()
    return docs


def test_pipeline_stage_graph_replay_equals_eager():
    eager = _device_run(False)
    replay = _device_run(True)
    assert eager == replay


def test_pipeline_stage_changes_no_other_output():
    scenes = _scenes()[:4]
    a = _pipeline(map_json=True, maxhold=True)
    b = _pipeline(map_json=True)
    for i, (x, y) in enumerate(scenes):
        ra, rb = a.process(x, y), b.process(x, y)
        assert np.array_equal(ra["map"], rb["map"])
        assert ra["noisePower"] == rb["noisePower"] and ra["maxPower"] == rb["maxPower"]
        da, db = ra["detections"], rb["detections"]
        assert np.array_equal(da.delay, db.delay) and np.array_equal(da.doppler, db.doppler)
        assert np.array_equal(da.snr, db.snr)
        assert a.fetch_map_json(i) == b.fetch_map_json(i)
