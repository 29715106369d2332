"""GPU: pipelines driven as bench.py drives them -- several CPIs in flight, on streams the caller owns -- against a
serial run of the same CPIs (a fresh pipeline, one CPI per submit -> fetch), bit for bit.

Every CPI of a pipeline shares its buffers (the filtered channel, the CAF scratch, the detection list, the status
word), so a fetch, or a submit on another stream, must run after the pipeline's last CPI whatever stream it went on.
The ordering tests put a bounded backlog (torch.cuda._sleep) on the submit stream and check that the CPI under test
has not started when the call under test is made, so the ordering is exercised every time, not by chance."""
import json
import struct

import numpy as np
import pytest
import torch

import bench
from blah2_b200.process import Pipeline
from blah2_b200.scene import make_scene
from cpi_products import code, cpi_products
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

FS, N = 200000, 40000
SMALL = (-5, 60, -500, 500, FS, N)
CLUTTER = (-5, 30)
DET = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
TRK = dict(M=2, N=3, delete=4, maxAcc=30, fc=204640000)
METRICS = (0.0, -1.005, 1e21)
T0 = 1731000000000
BACKLOG_CYCLES = 120_000_000  # 60 ms at the H100's 1.98 GHz boost clock, longer at lower clocks
NPIPE, NB = 6, 10             # bench.py's pipelines per GPU and rotated input sets
BENCH_PIPE = dict(clutter=bench.CLUTTER, detection=bench.DET, device=0)


def _pipeline(spectrum=True):
    """The small geometry with every stage on; without `spectrum`, no spectrum and IQ-data stages (submit_map then
    needs no spectrum parts)."""
    kw = dict(spectrum_bandwidth=2000) if spectrum else {}
    p = Pipeline(*SMALL, roundHamming=True, clutter=CLUTTER, detection=DET, device=0, map_json=True, maxhold=True,
                 detection_json=True, max_held_detections=1 << 16, tracker=TRK, max_track_history=32, **kw)
    if spectrum:
        p.enable_iqdata_json(*METRICS)
    p.enable_timing_json(T0)
    return p


def _small_inputs():
    """Three distinct CPIs of the small geometry as complex128 host arrays, and one whose reference channel is zero:
    its clutter-filter solve fails."""
    sc = make_scene(N, FS, seed=20261019)
    cpis = [(np.roll(sc.x, 977 * b), np.roll(sc.y, 977 * b)) for b in range(3)]
    return cpis + [(np.zeros(N, complex), sc.y)]


def _dev(z):
    return torch.from_numpy(np.ascontiguousarray(z).astype(np.complex64)).cuda()


def _map_buf(pipe):
    g = pipe.geometry
    return torch.full((g.n_doppler_bins, g.n_delay_bins), float("nan"), dtype=torch.complex64, device="cuda")


def _fetch(pipe, stream=None):
    """Pipeline.fetch(stream) as bytes: (skipped, noisePower and maxPower, the detections' delay, Doppler, SNR)."""
    r = pipe.fetch(stream)
    d = r["detections"]
    return (r["skipped"], struct.pack("<2d", r["noisePower"], r["maxPower"]), d.delay.tobytes(), d.doppler.tobytes(),
            d.snr.tobytes())


def _timing_keys(doc):
    """The timing document's keys in order: its stage times come from the device clock."""
    return doc if not isinstance(doc, bytes) else list(json.loads(doc))


def _products(pipe, ts, stream=None):
    """The fetch on `stream`, every enabled fetch_* in blah2's order, and the timing document's keys."""
    out = dict(cpi_products(pipe, ts, fetch=lambda p: _fetch(p, stream)))
    out["timing"] = _timing_keys(code(lambda: pipe.fetch_timing_json(ts)))
    return out


def _backlog(stream):
    """A bounded spin on `stream`, then an event: the work enqueued after it cannot start for tens of ms."""
    with torch.cuda.stream(stream):
        torch.cuda._sleep(BACKLOG_CYCLES)
    ev = torch.cuda.Event()
    ev.record(stream)
    return ev


def _assert_pending(ev):
    assert not ev.query(), "inconclusive: the backlog finished before the call under test"


def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k] == b[k], k


# ---- 1a: a fetch orders itself after the CPI it fetches ------------------------------------------------------------

FETCH_KINDS = ["eager", "replay", "map", "failed"]


def _fetch_run(kind, backlog, fetch_on):
    """A prior CPI submitted and fetched on S, then the CPI under test submitted on S by `kind` and fetched on
    `fetch_on` ("S", "none" or "third"); behind a backlog on S when `backlog`.  Returns both CPIs' products and
    maps."""
    cpis = _small_inputs()
    pipe = _pipeline(spectrum=kind != "map")
    S, third = torch.cuda.Stream(), torch.cuda.Stream()
    prior, tested = cpis[0], cpis[3 if kind == "failed" else 1]
    xs = [_dev(prior[0]), _dev(tested[0])]
    ys = [_dev(prior[1]), _dev(tested[1])]
    maps = [_map_buf(pipe), _map_buf(pipe)]
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    if kind == "map":  # the maps submit_map takes, from a pipeline of the same geometry
        src = Pipeline(*SMALL, roundHamming=True, clutter=CLUTTER, detection=DET, device=0)
        mm = [_map_buf(pipe), _map_buf(pipe)]
        for i in range(2):
            src.submit_device(xs[i], ys[i], mm[i])
            assert not src.fetch()["skipped"]
        src.close()
    torch.cuda.synchronize()
    if kind == "replay":
        pipe.prepare_device(xs[1], ys[1], maps[1], S.cuda_stream)

    def submit(i):
        if kind == "map":
            pipe.submit_map(mm[i], status, stream=S.cuda_stream)
        else:
            pipe.submit_device(xs[i], ys[i], maps[i], S.cuda_stream)

    try:
        submit(0)
        first = _products(pipe, T0 + 1000, S.cuda_stream)
        ev = _backlog(S) if backlog else None
        submit(1)
        if ev is not None:
            _assert_pending(ev)
        st = {"S": S.cuda_stream, "none": None, "third": third.cuda_stream}[fetch_on]
        second = _products(pipe, T0 + 2000, st)
    finally:
        torch.cuda.synchronize()
    out = (first, second, [m.cpu() for m in (mm if kind == "map" else maps)])
    pipe.close()
    return out


@pytest.mark.parametrize("fetch_on", ["none", "third"])
@pytest.mark.parametrize("kind", FETCH_KINDS)
def test_fetch_waits_for_the_cpi_it_fetches(kind, fetch_on):
    ref_first, ref_second, ref_maps = _fetch_run(kind, False, "S")
    first, second, maps = _fetch_run(kind, True, fetch_on)
    assert ref_second["fetch"][0] == (kind == "failed")
    _same(first, ref_first)
    _same(second, ref_second)
    for a, b in zip(maps, ref_maps):
        assert torch.equal(a, b)


# ---- 1a: a submit on another stream orders itself after the unfetched CPI ------------------------------------------

SECOND_KINDS = ["device", "prepare", "failed", "host", "rspduo", "ci8", "cf32"]


def _ci8(z):
    b = np.empty((z.shape[0], 2), dtype=np.int8)
    b[:, 0], b[:, 1] = z.real, z.imag
    return b


def _int8_values(z):
    """z scaled and rounded into int8's range: the ci8 entry's samples, as complex128."""
    q = np.round(z * (100.0 / np.max(np.abs(np.concatenate([z.real, z.imag])))))
    return np.clip(q.real, -128, 127) + 1j * np.clip(q.imag, -128, 127)


def _host_args(kind, x, y):
    """The buffers host entry `kind` takes for the CPI (x, y), pinned."""
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    if kind == "host":
        return pin(x.astype(np.complex128)), pin(y.astype(np.complex128))
    if kind == "rspduo":
        iq = np.empty((x.shape[0], 4), dtype="<i2")
        iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = x.real, x.imag, y.real, y.imag
        return (pin(iq),)
    if kind == "ci8":
        return pin(_ci8(x)), pin(_ci8(y))
    return pin(x.astype(np.complex64)), pin(y.astype(np.complex64))


def _submit_host(pipe, kind, args, map_out):
    f = {"host": pipe.submit_host, "rspduo": pipe.submit_host_rspduo, "ci8": pipe.submit_host_ci8,
         "cf32": pipe.submit_host_cf32}[kind]
    f(*args, map_out=map_out)


def _second_run(kind, inflight):
    """CPI A submitted on S1 (behind a backlog when `inflight`), then CPI B of other inputs by `kind` on S2 (device
    kinds) or the pipeline's own stream (host kinds) with no fetch between; serially, A is fetched first.  After the
    device is idle, B is fetched.  Returns A's map, B's map (map_out for the host kinds) and B's products."""
    cpis = _small_inputs()
    pipe = _pipeline()
    S1, S2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = cpis[0]
    b = cpis[3] if kind == "failed" else cpis[1]
    if kind == "ci8":
        a, b = (_int8_values(a[0]), _int8_values(a[1])), (_int8_values(b[0]), _int8_values(b[1]))
    xa, ya, xb, yb = _dev(a[0]), _dev(a[1]), _dev(b[0]), _dev(b[1])
    ma, mb = _map_buf(pipe), _map_buf(pipe)
    host = kind in ("host", "rspduo", "ci8", "cf32")
    args = _host_args(kind, *b) if host else None
    g = pipe.geometry
    map_out = torch.full((g.n_doppler_bins, g.n_delay_bins), complex("nan"), dtype=torch.complex128).pin_memory()
    torch.cuda.synchronize()
    try:
        ev = _backlog(S1) if inflight else None
        pipe.submit_device(xa, ya, ma, S1.cuda_stream)
        if not inflight:
            pipe.fetch(S1.cuda_stream)
        if ev is not None:
            _assert_pending(ev)
        if host:
            _submit_host(pipe, kind, args, map_out)
        elif kind == "prepare":
            pipe.prepare_device(xb, yb, mb, S2.cuda_stream)
        else:
            pipe.submit_device(xb, yb, mb, S2.cuda_stream)
        torch.cuda.synchronize()  # A, which ran after B unless B waited for it, has finished
        out = (ma.cpu(), map_out.clone() if host else mb.cpu(),
               _products(pipe, T0 + 1000, None if host else S2.cuda_stream))
    finally:
        torch.cuda.synchronize()
    pipe.close()
    return out


@pytest.mark.parametrize("kind", SECOND_KINDS)
def test_submit_on_another_stream_waits_for_the_unfetched_cpi(kind):
    ref_a, ref_b, ref = _second_run(kind, False)
    ma, mb, got = _second_run(kind, True)
    assert ref["fetch"][0] == (kind == "failed")
    assert torch.equal(ma, ref_a)
    assert torch.equal(mb, ref_b) and not torch.isnan(torch.view_as_real(mb)).any()
    _same(got, ref)


# ---- 1b, 1c: bench.py's regimes, every CPI checked -----------------------------------------------------------------

@pytest.fixture(scope="module")
def bench_sets():
    """bench.py's scene and its 10 input sets on the device, and each set's serial map and fetch."""
    sc = make_scene(bench.N, bench.FS, seed=20260923)
    x0 = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    y0 = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    xs = [torch.roll(x0, 977 * b) for b in range(NB)]
    ys = [torch.roll(y0, 977 * b) for b in range(NB)]
    pipe = Pipeline(**bench.GEOM, **BENCH_PIPE)
    g = pipe.geometry
    maps, fetches = [], []
    for b in range(NB):
        m = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
        torch.cuda.synchronize()
        pipe.submit_device(xs[b], ys[b], m)
        fetches.append(_fetch(pipe))
        maps.append(m)
    pipe.close()
    return sc, xs, ys, maps, fetches


def test_serial_bench_cpi_equals_the_oracle(bench_sets, relerr, monkeypatch):
    """The serial reference itself, on input set 3: the map within 1e-5 of the FP64 oracle chain, the detection list
    the oracle's, as test_fullsize_gpu checks config 2."""
    monkeypatch.setenv("BLAH2_ORACLE_WORKERS", "-1")
    sc, _, _, maps, fetches = bench_sets
    geom = [bench.GEOM[k] for k in ("delayMin", "delayMax", "dopplerMin", "dopplerMax", "fs", "nSamples")]
    g = O.ambiguity_geometry(*geom, True)
    ref = O.chain(np.roll(sc.x, 977 * 3), np.roll(sc.y, 977 * 3), g, clutter=bench.CLUTTER, det=bench.DET)
    e = relerr(maps[3].cpu().numpy().astype(np.complex128), ref["map"])
    assert e[0] < 1e-5 and e[1] < 1e-5, e
    skipped, _, delay, doppler, snr = fetches[3]
    assert not skipped
    got = [np.frombuffer(v, dtype=np.float64) for v in (delay, doppler, snr)]
    assert len(got[0]) == len(ref["detections"][0]) > 0
    dop_res = bench.FS / bench.N
    assert np.max(np.abs(got[0] - ref["detections"][0])) < 1e-3
    assert np.max(np.abs(got[1] - ref["detections"][1])) < 1e-3 * dop_res + 1e-6
    assert np.max(np.abs(got[2] - ref["detections"][2])) < 1e-3


def _device_regime(bench_sets, n_cpis, slot_of, n_slots, n_prep):
    """bench.py's device loop: CPI i on pipeline i % 6 and its stream, input set i % 10, map slot slot_of(i), all
    n_cpis queued before any fetch, after graphs were prepared for the triples of CPIs 0 .. n_prep - 1 (none: every
    CPI eager).  Returns the slots, each pipeline's final fetch and its last CPI."""
    _, xs, ys, _, _ = bench_sets
    pipes = [Pipeline(**bench.GEOM, **BENCH_PIPE) for _ in range(NPIPE)]
    g = pipes[0].geometry
    ring = torch.full((n_slots, g.n_doppler_bins, g.n_delay_bins), float("nan"), dtype=torch.complex64, device="cuda")
    streams = [torch.cuda.Stream() for _ in range(NPIPE)]
    torch.cuda.synchronize()
    if n_prep:  # bench.py's plan creation
        for i in range(n_prep):
            p = i % NPIPE
            pipes[p].prepare_device(xs[i % NB], ys[i % NB], ring[slot_of(i)], streams[p].cuda_stream)
        ring.fill_(float("nan"))
        torch.cuda.synchronize()
    try:
        for i in range(n_cpis):
            p = i % NPIPE
            with torch.cuda.stream(streams[p]):
                pipes[p].submit_device(xs[i % NB], ys[i % NB], ring[slot_of(i)], streams[p].cuda_stream)
        finals = [_fetch(pipes[p], streams[p].cuda_stream) for p in reversed(range(NPIPE))][::-1]
    finally:
        torch.cuda.synchronize()
    last = [max(i for i in range(n_cpis) if i % NPIPE == p) for p in range(NPIPE)]
    for p in pipes:
        p.close()
    return ring, finals, last


@pytest.mark.parametrize("graph", [True, False], ids=["replay", "eager"])
def test_bench_device_regime_every_cpi(bench_sets, graph):
    """bench.py's multi-GPU ring layout: every CPI its own slot, six CPIs queued per pipeline.  CPIs i and i + 30 run
    the same input set on the same pipeline, so a replay must tell their graphs apart by the map slot."""
    maps, fetches = bench_sets[3], bench_sets[4]
    n = 6 * NPIPE
    ring, finals, last = _device_regime(bench_sets, n, lambda i: i, n, n if graph else 0)
    for i in range(n):
        assert torch.equal(ring[i], maps[i % NB]), i
    for p in range(NPIPE):
        assert finals[p] == fetches[last[p] % NB], p


def test_bench_one_gpu_layout(bench_sets):
    """bench.py's 1-GPU layout: slot i % 6, graphs prepared for all 60 (set, pipeline) pairs, 20 CPIs queued."""
    maps, fetches = bench_sets[3], bench_sets[4]
    ring, finals, last = _device_regime(bench_sets, 20, lambda i: i % NPIPE, NPIPE, NB * NPIPE)
    for p in range(NPIPE):
        assert torch.equal(ring[p], maps[last[p] % NB]), p
        assert finals[p] == fetches[last[p] % NB], p


@pytest.mark.parametrize("kind", ["host", "rspduo", "ci8", "cf32"])
def test_bench_end_to_end_regime(bench_sets, kind):
    """bench.py's e2e loop: six pipelines on their own streams, pinned inputs shared as hx[i % 2], one map_out per
    pipeline, the fetch of CPI i - 6 before each submit.  Every fetched CPI equals the serial run of its set."""
    sc = bench_sets[0]
    sets = []
    for b in range(2):
        x, y = np.roll(sc.x, 977 * b), np.roll(sc.y, 977 * b)
        if kind == "ci8":
            x, y = _int8_values(x), _int8_values(y)
        sets.append(_host_args(kind, x, y))
    pipes = [Pipeline(**bench.GEOM, **BENCH_PIPE) for _ in range(NPIPE)]
    g = pipes[0].geometry
    shape = (g.n_doppler_bins, g.n_delay_bins)
    serial = []
    for b in range(2):
        m = torch.empty(shape, dtype=torch.complex128).pin_memory()
        _submit_host(pipes[0], kind, sets[b], m)
        serial.append((_fetch(pipes[0]), m))
    hmaps = [torch.full(shape, complex("nan"), dtype=torch.complex128).pin_memory() for _ in range(NPIPE)]
    steps = 3 * NPIPE
    got = []
    try:
        for i in range(steps + NPIPE):
            p = i % NPIPE
            if i >= NPIPE:
                got.append((i - NPIPE, _fetch(pipes[p]), hmaps[p].clone()))
            if i < steps:
                _submit_host(pipes[p], kind, sets[i % 2], hmaps[p])
    finally:
        torch.cuda.synchronize()
    for p in pipes:
        p.close()
    assert len(got) == steps
    for i, f, m in got:
        ref_f, ref_m = serial[i % 2]
        assert f == ref_f, i
        assert torch.equal(m, ref_m), i
