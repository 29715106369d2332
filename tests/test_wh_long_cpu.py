"""CPU: the clutter filter above 2048 taps, without a GPU.

* The tap limit is 4096: 4097 and 5000 taps are rejected at create with "taps" in the error, before any device call.
* The long solve kernel's step bodies (blah2_b200/csrc/solve_steps.cuh) run on the CPU (tests/native/solve_long_sim.cu)
  at 2049 and 4096 taps against a dense long-double Cholesky: weights and "not positive definite" verdicts.
* The fixtures tests/golden/wh_long_*.npz (the reference's own a, b, w and y') agree with the numpy restatement.
"""
import ctypes as C
import glob
import os
import shutil
import subprocess

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.scene import make_scene
from oracle import blah2_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "wh_long_*.npz")))


@pytest.mark.parametrize("taps", [4097, 5000])
def test_more_than_4096_taps_are_rejected(taps):
    lib = capi.load()
    h = C.c_void_p()
    assert lib.b200dd_wh_create(-10, taps - 10, 1000000, -1, C.byref(h)) == capi.ERR_GEOMETRY
    assert b"taps" in lib.b200dd_last_error()
    assert lib.b200dd_wh_create_chunk(-10, taps - 10, 1000000, 0, 500000, -1, C.byref(h)) == capi.ERR_GEOMETRY
    assert b"taps" in lib.b200dd_last_error()


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="no nvcc")
def test_long_toeplitz_solve_host_simulation(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "solve_long_sim")
    subprocess.run([nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-o", exe,
                    os.path.join(ROOT, "tests", "native", "solve_long_sim.cu")], check=True, capture_output=True)
    r = subprocess.run([exe, "2049", "4096"], capture_output=True, text=True)
    assert r.returncode == 0 and "SOLVE_LONG_SIM OK" in r.stdout, r.stdout + r.stderr


def test_fixtures_cover_the_new_ranges():
    names = {os.path.basename(p)[8:-4] for p in FIXTURES}
    assert {"t2049", "t2050", "t2418", "t2419", "t3585", "t3586", "t4096", "t4096p", "fail4096"} <= names
    taps = {int(np.load(p)["delayMax"]) - int(np.load(p)["delayMin"]) for p in FIXTURES}
    assert min(taps) == 2049 and max(taps) == 4096
    dmins = [int(np.load(p)["delayMin"]) for p in FIXTURES]
    assert min(dmins) < 0 and 0 in dmins and max(dmins) > 0


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[8:-4] for p in FIXTURES])
def test_fixture_agrees_with_the_numpy_restatement(path, relerr):
    d = np.load(path)
    dm, dM, n, seed = int(d["delayMin"]), int(d["delayMax"]), int(d["N"]), int(d["seed"])
    sc = make_scene(n, 2000000, seed=4100 if seed < 0 else seed)
    x = np.zeros(n, dtype=np.complex128) if seed < 0 else sc.x
    ok, w, a, b, xs = O.wienerhopf_weights(x, sc.y, dm, dM)
    assert ok == bool(d["ok"])
    assert relerr(d["a"], a)[0] < 1e-12 if np.any(a) else not np.any(d["a"])
    assert relerr(d["b"], b)[0] < 1e-12 if np.any(b) else not np.any(d["b"])
    if not ok:
        return
    assert relerr(d["w"], w)[0] < 1e-12
    y = O.wienerhopf_apply(xs, sc.y, w)
    step = int(d["step"])
    assert relerr(d["sub"], y[::step])[0] < 1e-12
    assert abs(float(d["norm"]) - np.linalg.norm(y)) < 1e-12 * np.linalg.norm(y)
