"""CPU: the exact truth of tests/conditioned_cases.py, and the solve kernels' step bodies on ill-conditioned systems.

* The correlations of integer inputs are integers: the FP64 FFT sums are within 0.05 of them, and the rounded values
  equal int64 dot products at the spot-checked lags.
* The iteratively refined weights equal a 50-digit mpmath Levinson solve, and scipy's solve_toeplitz on white
  references; the exact output equals the oracle's FFT filter where the system is well conditioned.
* The split (1-448 taps) and long (2049-4096 taps) solve kernels' step bodies (blah2_b200/csrc/solve_steps.cuh, run on
  the CPU by tests/native/solve_{split,long}_sim.cu --system) solve the conditioned systems as accurately as the
  oracle's LAPACK Cholesky does: err(sim) <= 10 err(oracle) + 1e-13 against the exact weights, and against the exact
  filtered output y' except the listed known misses.
"""
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.linalg as sla

import conditioned_cases as CC
from oracle import blah2_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 100000
C_RATIO, FLOOR_W = 10.0, 1e-13
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
needs_nvcc = pytest.mark.skipif(not os.path.exists(NVCC), reason="no nvcc")


@functools.lru_cache(maxsize=None)
def scene(ref, scale):
    return CC.make_case_scene(ref, scale, N, seed=CC.scene_seed(ref, scale))


@functools.lru_cache(maxsize=None)
def system(ref, scale, dm, dM):
    """(a, b, exact w, cond, oracle w) of one scene and clutter window."""
    sc = scene(ref, scale)
    a, b, dist = CC.exact_correlations(sc.x, sc.y, dm, dM)
    assert dist < 0.05
    A = CC.toeplitz_matrix(a)
    cf = sla.cho_factor(A, lower=False)
    truth = CC.exact_weights(a, b, cf)
    ok, w_ref = O.wienerhopf_weights(sc.x, sc.y, dm, dM)[:2]
    assert ok
    return a, b, truth.w, CC.cond_estimate(A, cf), w_ref


def filtered(ref, scale, dm, w):
    """y' of the oracle's filter (WienerHopf.cpp:125-160) applied to the weights w."""
    sc = scene(ref, scale)
    return O.wienerhopf_apply(CC.shifted_reference(sc.x, dm), sc.y, w)


@functools.lru_cache(maxsize=None)
def exact_output(ref, scale, dm, dM):
    sc = scene(ref, scale)
    return CC.exact_output(sc.x, sc.y, dm, system(ref, scale, dm, dM)[2])


def _rel(got, ref):
    return float(np.max(np.abs(got - ref)) / np.max(np.abs(ref)))


ALL_SCENES = [(r[0], s) for r in CC.REFERENCES for s in CC.SCALES]


@pytest.mark.parametrize("ref,scale", ALL_SCENES, ids=[f"{r}_{s}" for r, s in ALL_SCENES])
def test_correlations_are_exact_integers(ref, scale):
    sc = scene(ref, scale)
    for dm, dM in ((-10, 400), (7, 40)):
        a, b, dist = CC.exact_correlations(sc.x, sc.y, dm, dM)
        print(f"CONDITIONING {ref}_{scale} taps{dM - dm} dmin{dm}: distance to the integers {dist:.2e}")
        assert dist < 0.05
        for k in (0, 1, 17, dM - dm - 1):
            ak, bk = CC.correlation_lag_int64(sc.x, sc.y, dm, k)
            assert ak == a[k] and bk == b[k], (k, ak, a[k], bk, b[k])
        # the oracle's unrounded sums are the same to FP64 rounding
        _, _, a_o, b_o, _ = O.wienerhopf_weights(sc.x, sc.y, dm, dM)
        assert _rel(a_o, a) < 1e-14 and _rel(b_o, b) < 1e-14


MP_CASES = [("white", "int16", -10, 23), ("occ2", "int16", -10, 23), ("occ10_dc", "int16", 3, 36),
            ("occ10_tone", "int16", -10, 23), ("occ10_dc", "int16", -10, 110), ("occ2", "int8", 0, 64)]


@pytest.mark.parametrize("ref,scale,dm,dM", MP_CASES, ids=[f"{c[0]}_{c[1]}_taps{c[3] - c[2]}" for c in MP_CASES])
def test_refinement_equals_a_50_digit_levinson(ref, scale, dm, dM):
    a, b, w, cond, w_ref = system(ref, scale, dm, dM)
    w_mp = CC.mp_levinson(a, b)
    e, e_ref = _rel(w, w_mp), _rel(w_ref, w_mp)
    print(f"CONDITIONING {ref}_{scale} taps{dM - dm} cond {cond:.1e}: refined {e:.2e}, LAPACK {e_ref:.2e}")
    assert e < 4e-16


@pytest.mark.parametrize("dm,dM", [(-10, 400), (5, 2053)])
def test_refinement_equals_solve_toeplitz_on_white_references(dm, dM):
    a, b, w, cond, _ = system("white", "int16", dm, dM)
    assert cond < 1e3
    assert _rel(w, sla.solve_toeplitz((np.conj(a), a), b)) < 1e-13


def test_exact_output_equals_the_oracle_filter_on_a_white_reference():
    sc = scene("white", "int16")
    a, b, w, _, _ = system("white", "int16", -10, 400)
    y_true = CC.exact_output(sc.x, sc.y, -10, w)
    y_o = O.wienerhopf_apply(CC.shifted_reference(sc.x, -10), sc.y, w)
    assert _rel(y_o, y_true) < 1e-13


@functools.lru_cache(maxsize=None)
def _sim(name, tmpdir):
    exe = os.path.join(tmpdir, name)
    subprocess.run([NVCC, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-o", exe,
                    os.path.join(ROOT, "tests", "native", name + ".cu")], check=True, capture_output=True)
    return exe


def sim_solve(name, tmpdir, a, b):
    """(verdict, w) of the kernel's step bodies on the CPU."""
    n = a.shape[0]
    fin, fout = os.path.join(tmpdir, "system.bin"), os.path.join(tmpdir, "w.bin")
    with open(fin, "wb") as f:
        np.array([n], dtype=np.int32).tofile(f)
        np.concatenate([a, b]).astype(np.complex128).tofile(f)
    r = subprocess.run([_sim(name, tmpdir), "--system", fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(fout, dtype=np.uint8)
    return bool(raw[:4].view(np.int32)[0]), raw[4:].view(np.complex128)


SIM_CASES = [(k, ref, scale, dm, dM) for ref, scale in [("white", "int16"), ("occ10", "int16"), ("occ2", "int16"),
                                                        ("occ10_dc", "int16"), ("occ10_tone", "int16"),
                                                        ("occ10_dc", "int8")]
             for k, dm, dM in [("solve_split_sim", -10, 23), ("solve_split_sim", -10, 400),
                               ("solve_split_sim", 5, 453), ("solve_long_sim", -10, 2039)]]
SIM_CASES += [("solve_long_sim", "occ10_dc", "int16", -50, 4046), ("solve_long_sim", "occ2", "int16", 9, 4105),
              ("solve_split_sim", "occ2", "int16", -10, 438), ("solve_long_sim", "occ2", "int16", -10, 4086)]
# y' further than 10x the oracle's error from the exact y' (the weights stay within their bar): the Schur / Levinson
# recursion is weakly stable (test_levinson_leaves_its_error_in_the_output)
KNOWN_SIM_Y = {
    ("solve_long_sim", "occ2", "int16", -10, 2039),     # 2049 taps, cond 1.4e10: y' 38x the oracle's error, w 4.6x
    ("solve_long_sim", "occ2", "int16", -10, 4086),     # 4096 taps, cond 3.3e10: y' 59x, w 5.1x
}


@needs_nvcc
@pytest.mark.parametrize("kind,ref,scale,dm,dM", SIM_CASES,
                         ids=[f"{c[0][6:-4]}_{c[1]}_{c[2]}_taps{c[4] - c[3]}_dmin{c[3]}" for c in SIM_CASES])
def test_step_bodies_on_conditioned_systems(kind, ref, scale, dm, dM, tmp_path_factory):
    """Weights always within the bar; y' (the oracle's filter applied to the simulation's weights) within it except
    the known misses of KNOWN_SIM_Y, which must still miss."""
    a, b, w, cond, w_ref = system(ref, scale, dm, dM)
    ok, w_sim = sim_solve(kind, str(tmp_path_factory.getbasetemp()), a, b)
    assert ok
    y = exact_output(ref, scale, dm, dM)
    e, e_ref = _rel(w_sim, w), _rel(w_ref, w)
    ey, ey_ref = _rel(filtered(ref, scale, dm, w_sim), y), _rel(filtered(ref, scale, dm, w_ref), y)
    print(f"CONDITIONING {kind} {ref}_{scale} taps{dM - dm} cond {cond:.1e}: w err {e:.2e}, oracle {e_ref:.2e}, "
          f"ratio {e / e_ref:.2f}; y' err {ey:.2e}, oracle {ey_ref:.2e}, ratio {ey / ey_ref:.2f}")
    assert e <= C_RATIO * e_ref + FLOOR_W
    y_ok = ey <= C_RATIO * ey_ref + FLOOR_W
    if (kind, ref, scale, dm, dM) in KNOWN_SIM_Y:
        assert not y_ok, "known y' miss now within the bar: drop it from KNOWN_SIM_Y"
        pytest.xfail(f"known y' miss: {ey:.2e} against the oracle's {ey_ref:.2e} (weakly stable recursion)")
    assert y_ok, (ey, ey_ref)


def test_levinson_leaves_its_error_in_the_output():
    """Why the solve kernels can miss the y' bar while their weights meet the w bar (KNOWN_SIM_Y,
    test_wh_conditioning_gpu.KNOWN_Y): a plain FP64 Levinson-Durbin solve (scipy's solve_toeplitz) of the 2 %-occupied
    system at 2048 taps is within ~100x of the oracle's weight error, but leaves its error where the reference channel
    has power: its y' error is over 1000x the backward-stable Cholesky's."""
    ref, scale, dm, dM = "occ2", "int16", -10, 2038
    a, b, w, cond, w_ref = system(ref, scale, dm, dM)
    w_lev = sla.solve_toeplitz((np.conj(a), a), b)
    y = exact_output(ref, scale, dm, dM)
    ey, ey_ref = _rel(filtered(ref, scale, dm, w_lev), y), _rel(filtered(ref, scale, dm, w_ref), y)
    e, e_ref = _rel(w_lev, w), _rel(w_ref, w)
    print(f"CONDITIONING levinson {ref}_{scale} taps{dM - dm} cond {cond:.1e}: w err {e:.2e} (oracle {e_ref:.2e}), "
          f"y' err {ey:.2e} (oracle {ey_ref:.2e}), y' ratio {ey / ey_ref:.0f}")
    assert ey > 1000 * ey_ref and ey / ey_ref > 10 * e / e_ref
