"""The detection tail's boundary cases (tests/det_cases.py) on the CPU: every tie is exact, the restatement is the
oracle and the compiled reference on every case, and every planted fault changes a list.

The same cases run on the device in tests/test_det_exact_gpu.py.
"""
import math
import os
import shutil
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import det_cases as D  # noqa: E402

from oracle import blah2_oracle as O  # noqa: E402
from oracle import refpath  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFAR_CASES = D.cfar_cases()
CENTROID_CASES = D.centroid_cases()
FLAGS = [(True, True), (True, False), (False, True), (False, False)]


def _cpu_values(m, noise, fused=False):
    return D.sq_values(m), D.db_values(D.log10_abs(m), noise, fused)


def _cfar(case, noise=D.NOISE, fault=None, fused=False):
    sq, db = _cpu_values(case["map"], noise, fused)
    p = case["params"]
    return D.cfar(sq, db, case["delay"], case["doppler"], p["pfa"], p["nGuard"], p["nTrain"], p["minDelay"],
                  p["minDoppler"], fault)


def _interp(case, flags, fault=None, fused=False, drop_fenced=False):
    db = D.db_values(D.log10_abs(case["map"]), case["noise"], fused)
    lst = case["list"]
    if drop_fenced:
        fenced = D.interpolate(*lst, db, case["delay"], case["doppler"], *flags)[3]
        lst = tuple(a[~fenced] if fenced.size == a.size else a for a in lst)
        assert not D.interpolate(*lst, db, case["delay"], case["doppler"], *flags)[3].any()
    return D.interpolate(*lst, db, case["delay"], case["doppler"], *flags, fault=fault)[:3], lst


def test_alpha_is_exact_for_power_of_two_windows():
    for n, a in D.ALPHA_EXACT.items():
        assert D.alpha(n, D.PFA) == a
        assert Fraction(a) == n * (Fraction(2) ** (16 // n) - 1)
        assert float(np.float32(a)) == a  # so only inexact alphas can tell a float table apart


def _threshold_exact(sqrow, j, nGuard, nTrain, pfa):
    """The threshold with every operation rounded on its own, in Fraction arithmetic."""
    left, right = D.train_cells(j, len(sqrow), nGuard, nTrain)
    n = len(left + right)
    s = Fraction(0)
    for k in left + right:
        s = Fraction(D.rn(s + Fraction(sqrow[k])))
    mean = Fraction(D.rn(s / n))
    return D.rn(Fraction(D.alpha(n, pfa)) * mean), s


@pytest.mark.parametrize("case", CFAR_CASES, ids=lambda c: c["name"])
def test_cfar_ties_are_exact(case):
    p = case["params"]
    nGuard, nTrain = D.int8(p["nGuard"]), D.int8(p["nTrain"])
    m = case["map"].real
    if case["f32"]:
        assert np.array_equal(m.astype(np.float32).astype(np.float64), m)
    for row, j, kind, T in case["ties"]:
        sqrow = [float(v) * float(v) for v in m[row]]
        # the real-valued cell's complex square is its square, and that square is exact for a float32 cell
        assert D.sq_values(case["map"][row:row + 1])[0].tolist() == sqrow
        if case["f32"]:
            assert all(Fraction(float(v)) ** 2 == Fraction(s) for v, s in zip(m[row], sqrow))
        Tx, _ = _threshold_exact(sqrow, j, nGuard, nTrain, p["pfa"])
        assert Tx == T == D.threshold(sqrow, j, nGuard, nTrain, p["pfa"])
        x = float(m[row][j])
        if kind == "at":  # the rounded square of a double cell, the exact square of a float32 one
            assert D.rn(Fraction(x) ** 2) == T and (Fraction(x) ** 2 == T or not case["f32"])
        elif kind == "below":
            assert sqrow[j] < T and math.nextafter(x, math.inf) ** 2 >= T or case["f32"]
        elif kind == "above":
            assert sqrow[j] > T
        else:  # between the sequential and the right-first sums
            Tr = D.threshold(sqrow, j, nGuard, nTrain, p["pfa"], "train_right_first")
            assert min(T, Tr) < sqrow[j] < max(T, Tr)


def test_cfar_cases_cover_every_window_size_and_the_mixed_sums():
    seen = set()
    for case in CFAR_CASES:
        if case["name"].startswith("edges_"):
            nDel = case["map"].shape[1]
            for j in range(nDel):
                seen.add(sum(map(len, D.train_cells(j, nDel, 1, 8))))
    assert seen == set(range(0, 17))
    # column 1: k = 0 lies in the left window's range and is excluded (CfarDetector1D.cpp:61)
    assert D.train_cells(1, 20, 0, 8)[0] == [] and D.train_cells(2, 20, 0, 8)[0] == [1]
    mixed = next(c for c in CFAR_CASES if c["name"] == "mixed_windows")
    kinds = {k for _, _, k, _ in mixed["ties"]}
    assert "between" in kinds and "at" in kinds
    for row, j, kind, T in mixed["ties"]:
        sqrow = [float(v) ** 2 for v in mixed["map"].real[row]]
        left, right = D.train_cells(j, len(sqrow), 2, 8)
        cells = [Fraction(sqrow[k]) for k in left + right]
        exact = D.rn(sum(cells) / 16 * 16)
        pair = list(cells)
        while len(pair) > 1:
            pair = [Fraction(D.rn(pair[i] + pair[i + 1])) for i in range(0, len(pair), 2)]
        alts = {D.threshold(sqrow, j, 2, 8, D.PFA, "train_right_first"), exact, D.rn(pair[0])}
        assert any(a != T for a in alts), "the sums agree: the case does not tell the orders apart"


@pytest.mark.parametrize("case", CFAR_CASES, ids=lambda c: c["name"])
def test_cfar_restatement_is_the_oracle(case):
    p = case["params"]
    got = _cfar(case)
    ref = O.cfar_1d(case["map"], case["delay"], case["doppler"], D.NOISE, p["pfa"], p["nGuard"], p["nTrain"],
                    p["minDelay"], p["minDoppler"])
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    # the oracle takes log10 from numpy, whose SIMD log10 may differ from the C library's by an ulp
    assert np.all(np.abs(got[2] - ref[2]) <= 4 * np.spacing(np.abs(ref[2]) + 16))
    nGuard = D.int8(p["nGuard"])
    for row, j, kind, T in case["ties"]:
        hit = any(d == j + case["delay"][0] and f == case["doppler"][row] for d, f in zip(got[0], got[1]))
        active = abs(case["doppler"][row]) >= p["minDoppler"] and case["delay"][j] >= D.int8(p["minDelay"])
        x = float(case["map"].real[row][j])
        assert hit == (active and x * x > T), (row, j, kind, nGuard)


@pytest.mark.parametrize("case", CENTROID_CASES, ids=lambda c: c[0])
def test_centroid_restatement_is_the_oracle(case):
    _, d, f, s = case
    P = D.CENTROID_PARAMS
    assert D.same(D.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"]),
                  O.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"]))


@pytest.mark.parametrize("flags", FLAGS)
def test_interpolate_restatement_is_the_oracle(flags):
    case = D.interp_case()
    got, lst = _interp(case, flags, drop_fenced=True)
    # the oracle divides Python floats and cannot evaluate the all-equal pattern's 0 / 0: compare it elsewhere
    ok = []
    for i in range(len(lst[0])):
        try:
            O.interpolate(*(a[i:i + 1] for a in lst), case["map"], case["delay"], case["doppler"], case["noise"], *flags)
            ok.append(i)
        except ZeroDivisionError:
            pass
    assert len(ok) >= len(lst[0]) - 1
    lst = tuple(a[ok] for a in lst)
    got = _interp(dict(case, list=lst), flags)[0]
    ref = O.interpolate(*lst, case["map"], case["delay"], case["doppler"], case["noise"], *flags)
    assert D.same(got, ref)


def test_interpolate_case_holds_its_patterns():
    case = D.interp_case()
    a, b = case["pair"]
    La, Lb = math.log10(a), math.log10(b)
    assert Lb < La and 10.0 * La == 10.0 * Lb
    assert D.fma(Lb, 10.0, -case["noise"]) < D.fma(La, 10.0, -case["noise"])
    out = D.interpolate(*case["list"], D.db_values(D.log10_abs(case["map"]), case["noise"]), case["delay"],
                        case["doppler"], True, True)
    assert np.isnan(out[2]).any()          # the all-equal pattern: 0 / 0 kept as NaN
    assert out[3].any()                    # the off-axis Doppler value reaches the fence


def _caught_by_cfar(fault):
    return [c["name"] for c in CFAR_CASES if not D.same(_cfar(c), _cfar(c, fault=fault))]


@pytest.mark.parametrize("fault", D.CFAR_FAULTS)
def test_cfar_cases_catch_planted_fault(fault):
    assert _caught_by_cfar(fault), fault


@pytest.mark.parametrize("fault", D.CENTROID_FAULTS)
def test_centroid_cases_catch_planted_fault(fault):
    P = D.CENTROID_PARAMS
    hit = [name for name, d, f, s in CENTROID_CASES
           if not D.same(D.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"]),
                         D.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"], fault))]
    assert hit, fault


@pytest.mark.parametrize("fault", D.INTERP_FAULTS)
def test_interpolate_case_catches_planted_fault(fault):
    case = D.interp_case()
    assert any(not D.same(_interp(case, fl)[0], _interp(case, fl, fault=fault)[0]) for fl in FLAGS), fault


def test_cases_catch_the_fused_db_value():
    """fma(log10|z|, 10, -noisePower) for the twice-rounded value: CFAR's SNRs change, and Interpolate drops the
    plateau pair's detection that the reference keeps."""
    assert any(not D.same(_cfar(c), _cfar(c, fused=True)) for c in CFAR_CASES)
    case = D.interp_case()
    for fl in [(True, False), (False, True)]:
        ref, fus = _interp(case, fl)[0], _interp(case, fl, fused=True)[0]
        assert len(fus[0]) < len(ref[0]), fl


@pytest.mark.skipif(not refpath.available(), reason="the compiled reference (oracle/_ref) is not built")
def test_compiled_reference_agrees_bit_for_bit():
    for case in CFAR_CASES:
        p = case["params"]
        ref = refpath.cfar_1d(case["map"], case["delay"], case["doppler"], D.NOISE, p["pfa"], p["nGuard"],
                              p["nTrain"], p["minDelay"], p["minDoppler"])
        assert D.same(_cfar(case), ref), case["name"]
    P = D.CENTROID_PARAMS
    for name, d, f, s in CENTROID_CASES:
        assert D.same(D.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"]),
                      refpath.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"])), name
    case = D.interp_case()
    for fl in FLAGS:
        got, lst = _interp(case, fl, drop_fenced=True)
        assert D.same(got, refpath.interpolate(*lst, case["map"], case["delay"], case["doppler"], case["noise"],
                                               *fl)), fl


def test_fused_db_value_on_scene_maps():
    """How often the contracted fma(log10|z|, 10, -noisePower) differs from the reference's twice-rounded value on
    scene maps, and how often it changes Interpolate's list (glibc log10 on both sides)."""
    from blah2_b200.scene import Target, make_scene

    fs, n = 2000000, 200000
    geom = (-10, 120, -5000, 5000, fs, n, True)
    det = dict(pfa=1e-5, nGuard=2, nTrain=6, minDelay=5, minDoppler=15.0, nCentroid=6)
    g = O.ambiguity_geometry(*geom)
    cells = diff = runs = decisions = positions = 0
    for seed in (5, 6, 7):
        sc = make_scene(n, fs, seed=seed, targets=[Target(37, 3000.0, -30.0), Target(92, -2000.0, -35.0)])
        out = O.chain(sc.x, sc.y, g, clutter=(-10, 60), det=det)
        L = D.log10_abs(out["map"])
        ref, fus = D.db_values(L, out["noisePower"]), D.db_values(L, out["noisePower"], fused=True)
        cells += L.size
        diff += int(np.sum(ref != fus))
        lst = out["centroid"]
        r = D.interpolate(*lst, ref, g.delay, g.doppler)
        f = D.interpolate(*lst, fus, g.delay, g.doppler)
        runs += len(lst[0])
        decisions += int(len(r[0]) != len(f[0]))
        if len(r[0]) == len(f[0]):
            positions += int(np.sum((r[0] != f[0]) | (r[1] != f[1])))
    frac = diff / cells
    print(f"fused dB value differs in {diff} of {cells} scene cells ({100 * frac:.1f} %); Interpolate: "
          f"{decisions} list-length changes and {positions} moved positions over {runs} detections")
    assert frac > 0.25


def _cuobjdump():
    c = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return c if os.path.exists(c) else None


@pytest.mark.skipif(_cuobjdump() is None or not os.path.exists(os.path.join(ROOT, "blah2_b200", "lib", "obj", "det.o")),
                    reason="needs the built detection object and cuobjdump")
def test_no_fused_db_value_in_the_detection_kernels():
    """Every dB value is 10 log10|z| - noisePower rounded twice: no DFMA with the immediate 10 in det.cu's SASS."""
    import re
    sass = subprocess.run([_cuobjdump(), "-sass", os.path.join(ROOT, "blah2_b200", "lib", "obj", "det.o")],
                          capture_output=True, text=True, check=True).stdout
    assert "Function" in sass
    fused = [ln.strip() for ln in sass.splitlines() if re.search(r"\bDFMA\s+R\d+,\s*-?R\d+,\s*10,", ln)]
    assert not fused, fused[:4]
