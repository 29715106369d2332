"""GPU parity: CUDA cross-ambiguity function (through the C ABI) vs the oracle.

Mirrors the reference's test/unit/process/ambiguity/TestAmbiguity.cpp (constructor
known answers, Process_Simple on random IQ) and extends it with numeric pins against
oracle/blah2_oracle.py (itself pinned to the compiled reference).  Tolerance is the
north star's: map within 1e-5 relative (max-abs and Frobenius), written below.
"""
import numpy as np
import pytest

from blah2_b200.process import Ambiguity
from blah2_b200.scene import make_scene, random_iq, Target
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

TOL = 1e-5

# (delayMin, delayMax, dopplerMin, dopplerMax, fs, n, roundHamming)
GEOMS = [
    (-3, 20, -50, 50, 10000, 4000, False),        # tiny, odd everything
    (0, 31, -20, 60, 10000, 5000, True),          # asymmetric Doppler window -> pre-rotation (A2)
    (2, 40, -30, 30, 10000, 3000, True),          # positive delayMin
    (-10, 120, -5000, 5000, 2000000, 200000, True),   # many Doppler bins (1001), short batches
    (-10, 300, -300, 300, 2000000, 1000000, False),   # the reference unit test geometry
    (-10, 300, -300, 300, 2000000, 1000000, True),
    (0, 299, -128, 128, 2000000, 2000000, True),      # BASELINE config 1/2 geometry
    (-40, 1200, -100, 100, 2000000, 400000, True),    # wide delay window (nDel = 1241)
]


def _run(geom, x, y):
    amb = Ambiguity(*geom)
    m = amb.process(x, y)
    return amb, m


@pytest.mark.parametrize("geom", GEOMS)
def test_geometry_matches_reference_constructor(geom):
    amb = Ambiguity(*geom)
    g = O.ambiguity_geometry(*geom)
    assert amb.get_n_delay_bins() == g.nDelayBins
    assert amb.get_n_doppler_bins() == g.nDopplerBins
    assert amb.get_n_corr() == g.nCorr
    assert amb.get_nfft() == g.nfft
    assert amb.get_cpi() == g.cpi
    assert amb.get_doppler_middle() == g.dopplerMiddle
    assert np.array_equal(amb.delay, g.delay)
    assert np.array_equal(amb.doppler, g.doppler)


def test_constructor_known_answers():
    # TestAmbiguity.cpp:73-116
    a = Ambiguity(-10, 300, -300, 300, 2000000, 1000000)
    assert (a.get_n_corr(), a.get_n_delay_bins(), a.get_n_doppler_bins(), a.get_nfft()) == (3322, 311, 301, 6643)
    assert abs(a.get_cpi() - 0.5) < 0.02 and a.get_doppler_middle() == 0
    b = Ambiguity(-10, 300, -300, 300, 2000000, 1000000, True)
    assert b.get_nfft() == 6750


@pytest.mark.parametrize("geom", GEOMS)
def test_map_matches_oracle_random_iq(geom, relerr):
    n = geom[5]
    x, y = random_iq(n, seed=11)
    amb, m = _run(geom, x, y)
    g = O.ambiguity_geometry(*geom)
    ref, lx, ly = O.ambiguity_process(x, y, g)
    # range matrix first (localises a failure to K1 or K2)
    Rref = O.range_matrix(O.ambiguity_prerotate(np.asarray(x, np.complex128), g), np.asarray(y, np.complex128), g)
    e_r = relerr(amb.debug_range_matrix(), Rref)
    assert e_r[0] < TOL and e_r[1] < TOL, f"range matrix {e_r}"
    e = relerr(m.data, ref)
    assert e[0] < TOL and e[1] < TOL, f"map {e}"
    # Process_Simple assertions (TestAmbiguity.cpp:142-143) + metric parity within 1e-3 dB
    noise, mx = O.set_metrics(m.data)
    noise_ref, mx_ref = O.set_metrics(ref)
    assert mx > 0 and noise > 0
    assert abs(noise - noise_ref) < 1e-3 and abs(mx - mx_ref) < 1e-3
    assert amb.get_n_samples() == g.n_used


def test_map_matches_oracle_radar_scene(relerr):
    geom = (0, 299, -128, 128, 2000000, 2000000, True)
    sc = make_scene(geom[5], geom[4], seed=20260924)
    amb, m = _run(geom, sc.x, sc.y)
    g = O.ambiguity_geometry(*geom)
    ref, _, _ = O.ambiguity_process(sc.x, sc.y, g)
    e = relerr(m.data, ref)
    assert e[0] < TOL and e[1] < TOL, f"map {e}"
    # the targets must show up where they were put
    k = np.unravel_index(np.argmax(np.abs(m.data[:, 20:]) * (np.abs(m.doppler) > 20)[:, None]), m.data[:, 20:].shape)
    assert (k[1] + 20) in (37, 92, 151, 230)


@pytest.mark.parametrize("log2m", [8, 9, 10, 11, 12, 13])
def test_every_range_fft_length_gives_the_same_map(log2m, relerr, monkeypatch):
    monkeypatch.setenv("B200DD_CAF_LOG2M", str(log2m))
    geom = (-5, 60, -200, 200, 100000, 100000, True)
    x, y = random_iq(geom[5], seed=5)
    amb, m = _run(geom, x, y)
    assert amb.geometry.range_fft_len == (1 << log2m)
    g = O.ambiguity_geometry(*geom)
    ref, _, _ = O.ambiguity_process(x, y, g)
    e = relerr(m.data, ref)
    assert e[0] < TOL and e[1] < TOL, f"log2m={log2m} map {e}"


@pytest.mark.parametrize("log2m,parts", [(9, 1), (9, 2), (9, 3), (9, 100), (10, 2), (10, 3), (11, 100), (12, 2)])
def test_batch_split_into_parts_gives_the_same_map(log2m, parts, relerr, monkeypatch):
    """B200DD_CAF_PARTS: a batch's segments split over several CTAs, whose partial range matrices the Doppler kernel
    adds in a fixed order.  Same map and same range matrix as the oracle; more parts than segments are clamped."""
    monkeypatch.setenv("B200DD_CAF_LOG2M", str(log2m))
    monkeypatch.setenv("B200DD_CAF_PARTS", str(parts))
    geom = (-5, 60, -20, 20, 100000, 100000, True)       # nCorr 2439: 6 (M=512), 3 (1024), 2 (2048) segments
    if log2m == 12:
        geom = (-5, 60, -5, 5, 100000, 100000, True)     # nCorr 9090: 3 segments at M = 4096
    x, y = random_iq(geom[5], seed=6)
    amb, m = _run(geom, x, y)
    g = amb.geometry
    assert g.range_fft_len == (1 << log2m)
    assert g.range_segments > 1 and g.range_parts == min(parts, g.range_segments)
    og = O.ambiguity_geometry(*geom)
    ref, _, _ = O.ambiguity_process(x, y, og)
    e = relerr(m.data, ref)
    assert e[0] < TOL and e[1] < TOL, f"log2m={log2m} parts={parts} map {e}"
    Rref = O.range_matrix(np.asarray(x, np.complex128), np.asarray(y, np.complex128), og)
    assert relerr(amb.debug_range_matrix(), Rref)[0] < TOL
    # deterministic: the parts are added in a fixed order
    _, m2 = _run(geom, x, y)
    assert np.array_equal(m.data, m2.data)


def test_linearity_and_determinism_full_size():
    """Size-independent properties at BASELINE config-3 size (oracle too slow to run in
    seconds): CAF(x, a*y1 + b*y2) = a CAF(x,y1) + b CAF(x,y2), and bitwise repeatability."""
    geom = (0, 511, -256, 256, 10000000, 20000000, True)
    amb = Ambiguity(*geom)
    n = geom[5]
    rng = np.random.default_rng(3)
    x = (rng.integers(-2000, 2000, n) + 1j * rng.integers(-2000, 2000, n)).astype(np.complex128)
    y1 = (rng.integers(-2000, 2000, n) + 1j * rng.integers(-2000, 2000, n)).astype(np.complex128)
    y2 = np.roll(x, 100) * 0.25
    m1 = amb.process(x, y1).data
    m2 = amb.process(x, y2).data
    m12 = amb.process(x, 2.0 * y1 - 3.0 * y2).data
    lin = 2.0 * m1 - 3.0 * m2
    assert np.max(np.abs(m12 - lin)) / np.max(np.abs(lin)) < TOL
    again = amb.process(x, y1).data
    assert np.array_equal(again, m1)
    # y2 is x delayed by 100 bins: the zero-Doppler row must peak at delay bin 100
    zero = (amb.get_n_doppler_bins() - 1) // 2
    assert int(np.argmax(np.abs(m2[zero]))) == 100


def test_too_few_samples_is_an_error():
    from blah2_b200 import capi
    amb = Ambiguity(-3, 20, -50, 50, 10000, 4000)
    with pytest.raises(capi.B200ddError):
        amb.process(np.zeros(100, complex), np.zeros(100, complex))


def test_stagewise_entry_points_emulating_two_ranks(relerr):
    """b200dd_caf_range_device / b200dd_caf_doppler_device (single CPI split over GPUs, BASELINE config 5):
    two 'ranks' emulated on one device must reproduce the one-shot map bit for bit."""
    import torch
    from blah2_b200.shard import block_range, caf_single_cpi_sharded
    geom = (-5, 60, -200, 200, 100000, 100000, True)
    x, y = random_iq(geom[5], seed=12)
    amb = Ambiguity(*geom)
    g = amb.geometry
    dx = torch.from_numpy(x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(y.astype(np.complex64)).cuda()
    full = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        amb.process_device(dx, dy, full, s.cuda_stream)
        one = caf_single_cpi_sharded(amb, dx[: g.n_used], dy[: g.n_used], 0, 1, s)
        R = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
        for r in range(2):
            b0, nb = block_range(g.n_doppler_bins, r, 2)
            lo, hi = b0 * g.n_corr, (b0 + nb) * g.n_corr
            amb.range_device(dx[lo:hi], dy[lo:hi], b0, nb, R[b0:b0 + nb], s.cuda_stream)
        tiles = []
        for r in range(2):
            c0, nc = block_range(g.n_delay_bins, r, 2)
            t = torch.empty((g.n_doppler_bins, nc), dtype=torch.complex64, device="cuda")
            amb.doppler_device(R, c0, nc, t, s.cuda_stream)
            tiles.append(t)
    s.synchronize()
    assert torch.equal(one, full)
    assert torch.equal(torch.cat(tiles, dim=1), full)
    ref, _, _ = O.ambiguity_process(x, y, O.ambiguity_geometry(*geom))
    assert relerr(full.cpu().numpy().astype(np.complex128), ref)[0] < TOL


def test_single_cpi_plan_with_filter_on_one_gpu_matches_the_pipeline(relerr):
    """blah2_b200.shard.SingleCpiPlan (config-5 orchestration: chunked clutter filter + stage-wise CAF over the C-ABI
    communicator) at world size 1 must reproduce the ordinary whole-CPI path and the oracle."""
    import torch
    from blah2_b200.process import WienerHopfChunk
    from blah2_b200.shard import Comm, SingleCpiPlan
    from blah2_b200.scene import make_scene
    geom = (-5, 60, -200, 200, 100000, 100000, True)
    clutter = (-4, 40)
    sc = make_scene(geom[5], geom[4], seed=21, n_clutter=8)
    x = sc.x.astype(np.complex64)
    y = sc.y.astype(np.complex64)
    comm = Comm(0, 1, torch.cuda.current_device())
    amb = Ambiguity(*geom)
    plan = SingleCpiPlan(comm, amb, geom[5], torch.device("cuda"), clutter=clutter,
                         whc_factory=lambda a, b, n, c0, nc: WienerHopfChunk(a, b, n, c0, nc))
    plan.x_own.copy_(torch.from_numpy(x))
    plan.y_own.copy_(torch.from_numpy(y))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        m = plan.run(s)
    s.synchronize()
    assert plan.whc.last_status()
    ok, yf = O.wienerhopf_process(x.astype(np.complex128), y.astype(np.complex128), *clutter)
    ref, _, _ = O.ambiguity_process(x.astype(np.complex128), yf.astype(np.complex64).astype(np.complex128), O.ambiguity_geometry(*geom))
    e = relerr(m.cpu().numpy().astype(np.complex128), ref)
    assert ok and e[0] < TOL and e[1] < TOL, e
    comm.close()


@pytest.mark.parametrize("n_tiles", [1, 2, 3, 8])
def test_tile_placement_kernel_rebuilds_the_map(n_tiles):
    """b200dd_caf_place_tiles_device: the gathered delay-column tiles of an equal split (shard.block_range), stored back
    to back, become the row-major map in one kernel; b200dd_caf_place_tile_device does the same tile by tile."""
    import torch
    from blah2_b200.shard import block_range
    amb = Ambiguity(-5, 60, -200, 200, 100000, 100000, True)
    g = amb.geometry
    ref = torch.randn((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    cols = [block_range(g.n_delay_bins, r, n_tiles) for r in range(n_tiles)]
    tiles = torch.cat([ref[:, c0:c0 + nc].contiguous().reshape(-1) for c0, nc in cols])
    out = torch.zeros_like(ref)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        amb.place_tiles(tiles, n_tiles, out, s.cuda_stream)
    s.synchronize()
    assert torch.equal(out, ref)
    out2 = torch.zeros_like(ref)
    off = 0
    with torch.cuda.stream(s):
        for c0, nc in cols:
            amb.place_tile(tiles[off:off + g.n_doppler_bins * nc], c0, nc, out2, s.cuda_stream)
            off += g.n_doppler_bins * nc
    s.synchronize()
    assert torch.equal(out2, ref)
