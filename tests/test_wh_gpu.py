"""GPU parity: CUDA Wiener-Hopf clutter canceller (through the C ABI) vs the oracle.

The reference has NO test for WienerHopf (SURVEY.md s4), so the pins are the oracle
(oracle/blah2_oracle.py, itself checked against the compiled reference source + the
Armadillo/LAPACK restatement) and size-independent properties.
"""
import numpy as np
import pytest

from blah2_b200.process import Ambiguity, WienerHopf
from blah2_b200.scene import make_scene, Target
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

# (n, delayMin, delayMax, seed)
CASES = [
    (5000, -3, 20, 1),
    (20011, -10, 40, 2),        # prime-ish length: segments do not divide N
    (65536, 0, 100, 3),         # delayMin = 0
    (200000, -10, 400, 4),      # the reference's default clutter window (config/config.yml:29-32)
    (100000, 2, 60, 5),         # delayMin > 0 (reference's uint32 wrap semantics)
    (300000, -10, 1200, 6),     # many taps -> longer FFT plan, generic solve kernel (two rows per thread)
    (150000, -10, 700, 7),      # 710 taps: short-path solve kernel with the 1024-thread bound
    (400000, -10, 2030, 8),     # the largest supported system (2040 taps)
    (4096, 0, 1, 9),            # a single tap
]


def _scene(n, seed):
    return make_scene(n, 2e6, seed=seed, targets=[Target(25, 300.0, -40.0)])


@pytest.mark.parametrize("case", CASES)
def test_filter_matches_oracle_fp64_host_path(case, relerr):
    n, dm, dM, seed = case
    sc = _scene(n, seed)
    wh = WienerHopf(dm, dM, n)
    ok, y = wh.process(sc.x, sc.y)
    ok_ref, w_ref, a_ref, b_ref, xs = O.wienerhopf_weights(sc.x, sc.y, dm, dM)
    assert ok and ok_ref
    w, a, b = wh.debug_weights()
    assert relerr(a, a_ref)[0] < 1e-12, "auto-correlation"
    assert relerr(b, b_ref)[0] < 1e-12, "cross-correlation"
    assert relerr(w, w_ref)[0] < 1e-9, "weights"
    y_ref = O.wienerhopf_apply(xs, sc.y, w_ref)
    e = relerr(y, y_ref)
    assert e[0] < 1e-9 and e[1] < 1e-9, f"filtered surveillance {e}"
    # it must actually cancel clutter (when the tap window covers the direct path at lag 0)
    # (a single tap cannot: the scene's clutter is spread over several lags)
    if dm <= 0 and dM - dm >= 20:
        assert np.linalg.norm(y) < 0.1 * np.linalg.norm(sc.y)


def test_cholesky_failure_leaves_y_untouched():
    n = 4096
    wh = WienerHopf(-2, 10, n)
    y0 = np.ones(n, dtype=np.complex128) * (1 + 2j)
    ok, y = wh.process(np.zeros(n, dtype=np.complex128), y0)   # A = 0 -> not positive definite
    assert not ok
    assert np.array_equal(y, y0)
    assert not O.wienerhopf_process(np.zeros(n), y0, -2, 10)[0]


def test_device_path_complex64(relerr):
    import torch
    n, dm, dM = 200000, -10, 400
    sc = _scene(n, 7)
    wh = WienerHopf(dm, dM, n)
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    out = torch.empty_like(dy)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        wh.process_device(dx, dy, out, s.cuda_stream)
    s.synchronize()
    assert wh.last_status()
    ok, y_ref = O.wienerhopf_process(sc.x, sc.y, dm, dM)
    e = relerr(out.cpu().numpy().astype(np.complex128), y_ref)
    assert e[0] < 1e-6 and e[1] < 1e-6, f"{e}"   # float32 rounding of the output only
    # in-place (d_y_out aliasing d_y)
    with torch.cuda.stream(s):
        wh.process_device(dx, dy, dy, s.cuda_stream)
    s.synchronize()
    assert torch.equal(dy, out)


def test_clutter_filter_then_ambiguity_map_matches_oracle(relerr):
    """BASELINE config 2 shape at reduced size: WienerHopf -> Ambiguity, map within 1e-5."""
    fs, n = 2000000, 400000
    geom = (-10, 120, -300, 300, fs, n, True)
    sc = make_scene(n, fs, seed=9, targets=[Target(37, 110.0, -50.0), Target(92, -205.0, -55.0)])
    wh = WienerHopf(-10, 60, n)
    ok, yf = wh.process(sc.x, sc.y)
    assert ok
    m = Ambiguity(*geom).process(sc.x, yf)
    g = O.ambiguity_geometry(*geom)
    out = O.chain(sc.x, sc.y, g, clutter=(-10, 60))
    e = relerr(m.data, out["map"])
    assert e[0] < 1e-5 and e[1] < 1e-5, f"{e}"


def test_full_size_config2_against_oracle(relerr):
    """N = 2e6, 410 taps: the oracle still finishes in seconds at this size."""
    fs, n = 2000000, 2000000
    sc = make_scene(n, fs, seed=20260923)
    wh = WienerHopf(-10, 400, n)
    ok, y = wh.process(sc.x, sc.y)
    ok_ref, y_ref = O.wienerhopf_process(sc.x, sc.y, -10, 400)
    assert ok and ok_ref
    e = relerr(y, y_ref)
    assert e[0] < 1e-9 and e[1] < 1e-9, f"{e}"


def test_linearity_in_y_for_fixed_weights_property():
    """Idempotence-style property: filtering an already clutter-free y (pure noise,
    uncorrelated with x) changes it by at most the estimation noise of w."""
    n = 500000
    rng = np.random.default_rng(1)
    x = np.round(rng.standard_normal(n) * 1000) + 1j * np.round(rng.standard_normal(n) * 1000)
    y = np.round(rng.standard_normal(n) * 30) + 1j * np.round(rng.standard_normal(n) * 30)
    ok, yf = WienerHopf(-5, 100, n).process(x, y)
    assert ok
    assert np.linalg.norm(yf - y) < 0.05 * np.linalg.norm(y)


@pytest.mark.parametrize("log2m", [9, 10, 11, 12])
def test_every_fft_plan_gives_the_same_filter(log2m, relerr, monkeypatch):
    """Every FFT length of the FP64 kernels (B200DD_WH_LOG2M): middle radix 2, 4, 8, 16 of the DIT plan."""
    radix = 16
    monkeypatch.setenv("B200DD_WH_LOG2M", str(log2m))
    n, dm, dM = 50021, -5, 70
    sc = _scene(n, 13)
    wh = WienerHopf(dm, dM, n)
    ok, y = wh.process(sc.x, sc.y)
    ok_ref, y_ref = O.wienerhopf_process(sc.x, sc.y, dm, dM)
    assert ok and ok_ref
    e = relerr(y, y_ref)
    assert e[0] < 1e-9 and e[1] < 1e-9, f"radix {radix} M=2^{log2m}: {e}"


# (n, delayMin, delayMax, seed): one tap, 33, 50, 410 (the reference's), 448 and 510 taps, then every solve kernel at both
# ends of the tap range that picks it
@pytest.mark.parametrize("case", [(20011, -10, 40, 2), (200000, -10, 400, 4), (150000, 0, 1, 5), (150000, -3, 30, 6),
                                  (200000, -10, 438, 7), (200000, -10, 500, 8)]
                         + [(100000, -10, nb - 10, nb) for nb in (449, 480, 481, 992, 993, 1024, 1025, 2048)])
def test_all_solve_kernels_give_the_same_weights(case, relerr):
    """The tap count picks the solve kernel: split producer / consumer (1-448 taps), one-barrier-per-step short kernel
    with a 512- (449-480) or 1024-thread bound (481-992), generic kernel with one (993-1024) or two rows per thread
    (1025-2048).  On the correlation sums of a scene every kernel gives the weights LAPACK gives for the kernel's own
    Toeplitz system toeplitz(conj(a), a) w = b."""
    import scipy.linalg as sla
    n, dm, dM, seed = case
    sc = _scene(n, seed)
    wh = WienerHopf(dm, dM, n)
    ok, _ = wh.process(sc.x, sc.y)
    assert ok
    w, a, b = wh.debug_weights()
    assert relerr(w, np.linalg.solve(sla.toeplitz(np.conj(a), a), b))[0] < 1e-10


def _ar_sequence(nb, seed, pole=0.9):
    """First column a[k] of a Hermitian positive-definite Toeplitz matrix: the autocorrelation of a few complex AR(1) lines."""
    rng = np.random.default_rng(seed)
    k = np.arange(nb)
    a = np.zeros(nb, dtype=np.complex128)
    for _ in range(4):
        a += rng.uniform(0.5, 2.0) * (pole * rng.uniform(0.5, 1.0) * np.exp(2j * np.pi * rng.uniform())) ** k
    a[0] = a[0].real * 1.01
    return a


# every solve kernel at both ends of its tap range (1-448, 449-480, 481-992, 993-1024, 1025-2048), each with a
# first-pivot, early, mid-recursion and last-pivot failure
_SOLVE_ENDS = [(nb, bad) for nb in (449, 480, 481, 992, 993, 1024, 1025, 2048)
               for bad in (None, 0, 1, nb // 2, nb - 1) if (nb, bad) not in ((480, None), (480, 479))]


@pytest.mark.parametrize("nb,bad_at", [(1, None), (1, 0), (32, None), (33, None), (33, 1), (33, 20), (64, None), (65, 33),
                                       (410, None), (410, 1), (410, 30), (410, 31), (410, 215), (410, 409),
                                       (448, None), (448, 0), (448, 1), (448, 224), (448, 447), (480, None), (480, 479),
                                       (496, None), (496, 495), (600, 300), (710, None), (1210, None)] + _SOLVE_ENDS)
@pytest.mark.parametrize("mode", [(40000, 0), (120000, 0), (120000, 80000)])
def test_solve_kernels_on_given_toeplitz_systems(nb, bad_at, mode, relerr):
    """The solve kernel the tap count picks, on correlation sums handed in through the chunk API
    (b200dd_wh_chunk_filter_device): weights against LAPACK on the matrix the reference builds (WienerHopf.cpp:85-97),
    and the 'not positive definite' verdict -- WienerHopf.cpp:111-117: chol() fails -> process() returns false, y
    untouched -- when the leading minor of order bad_at + 1 is the first indefinite one (first pivot / early /
    mid-recursion / last pivot).  mode = (signal length, first sample) of the handle's 40000-sample chunk: the whole
    signal, its first or its last chunk (the pass-through of a failed CPI writes the chunk's own samples)."""
    import scipy.linalg as sla
    import torch
    from blah2_b200.process import WienerHopfChunk
    n = 40000
    n_total, c0 = mode
    a = _ar_sequence(nb, nb)
    rng = np.random.default_rng(nb + 1)
    b = rng.standard_normal(nb) + 1j * rng.standard_normal(nb)
    if bad_at == 0:
        a[0] = -1.0
    elif bad_at is not None:
        a[bad_at] = 3.0 * a[0]           # |a[k]| > a[0]: the minor of order k + 1 is indefinite, the smaller ones are not
    A = sla.toeplitz(np.conj(a), a)      # A(i,j) = a[j-i] (j >= i), conj(a[i-j]) (i > j)
    expect_ok = True
    try:
        np.linalg.cholesky(A)
    except np.linalg.LinAlgError:
        expect_ok = False
    assert expect_ok == (bad_at is None)
    if bad_at:
        np.linalg.cholesky(A[:bad_at, :bad_at])          # ... and it is the FIRST bad minor
    ch = WienerHopfChunk(0, nb, n_total, c0, n)
    xl, xr, yr = ch.halos()
    g = torch.Generator(device="cuda").manual_seed(5)
    x_loc = torch.view_as_complex(torch.randn((xl + n + xr, 2), device="cuda", generator=g))
    y_loc = torch.view_as_complex(torch.randn((n + yr, 2), device="cuda", generator=g))
    out = torch.full((n,), complex(7, 7), dtype=torch.complex64, device="cuda")
    ab = torch.from_numpy(np.concatenate([a, b])).cuda()
    ch.filter_device(ab, x_loc, y_loc, out)
    torch.cuda.synchronize()
    assert ch.last_status() == expect_ok
    if expect_ok:
        w = ch.debug_weights()[0]
        assert relerr(w, np.linalg.solve(A, b))[0] < 1e-10
    else:
        assert torch.equal(out, y_loc[:n])               # the surveillance channel passes through


@pytest.mark.parametrize("case", [(300000, -10, 400, 3, 7), (120000, 0, 60, 2, 8), (200003, -3, 129, 4, 9)])
def test_chunked_filter_emulating_several_ranks(case, relerr):
    """One CPI split over several GPUs (SURVEY.md s8e row 3), emulated on one device: every 'rank' correlates its
    chunk (right halo circular, as the reference's N-point correlations are), the partial (a, b) are summed, every
    rank solves the same system and filters its chunk (left halo = filter history, zero before sample 0).  The
    concatenated output must equal the one-GPU filter's and the oracle's."""
    import torch
    from blah2_b200.process import WienerHopfChunk
    from blah2_b200.shard import block_range
    n, dm, dM, world, seed = case
    sc = _scene(n, seed)
    xg = sc.x.astype(np.complex64)
    yg = sc.y.astype(np.complex64)
    wh = WienerHopf(dm, dM, n)
    dx, dy = torch.from_numpy(xg).cuda(), torch.from_numpy(yg).cuda()
    ref = torch.empty_like(dy)
    torch.cuda.synchronize()
    wh.process_device(dx, dy, ref)
    torch.cuda.synchronize()
    w_ref, a_ref, b_ref = wh.debug_weights()
    s = torch.cuda.Stream()
    chunks, ab_parts = [], []
    with torch.cuda.stream(s):
        for r in range(world):
            c0, nc = block_range(n, r, world)
            ch = WienerHopfChunk(dm, dM, n, c0, nc)
            xl, xr, yr = ch.halos()
            ix = (np.arange(c0 - xl, c0 + nc + xr)) % n          # (the first chunk's left halo is never used)
            iy = (np.arange(c0, c0 + nc + yr)) % n
            x_loc = torch.from_numpy(xg[ix]).cuda()
            y_loc = torch.from_numpy(yg[iy]).cuda()
            ab = torch.zeros(2 * ch.nBins, dtype=torch.complex128, device="cuda")
            ch.corr_device(x_loc, y_loc, ab, s.cuda_stream)
            chunks.append((ch, x_loc, y_loc, nc))
            ab_parts.append(ab)
        s.synchronize()
        ab_sum = torch.stack(ab_parts).sum(0)              # what the all-reduce over the ranks computes
        nb = chunks[0][0].nBins
        assert relerr(ab_sum[:nb].cpu().numpy(), a_ref)[0] < 1e-12 and relerr(ab_sum[nb:].cpu().numpy(), b_ref)[0] < 1e-12
        outs = []
        for ch, x_loc, y_loc, nc in chunks:
            o = torch.empty(nc, dtype=torch.complex64, device="cuda")
            ch.filter_device(ab_sum, x_loc, y_loc, o, s.cuda_stream)
            outs.append(o)
        s.synchronize()
    assert all(c[0].last_status() for c in chunks)
    got = torch.cat(outs).cpu().numpy()
    assert relerr(got, ref.cpu().numpy())[0] < 1e-6          # complex64 output rounding
    ok, y_ref = O.wienerhopf_process(xg.astype(np.complex128), yg.astype(np.complex128), dm, dM)
    assert ok and relerr(got, y_ref)[0] < 1e-6
