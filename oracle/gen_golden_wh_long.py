"""oracle/gen_golden_wh_long.py -- TEST INFRASTRUCTURE ONLY.

Fixtures of the clutter filter above 2048 taps, produced by the reference's UNMODIFIED WienerHopf::process
(oracle/_ref/libblah2whlong.so, oracle/whlong/) on seeded scenes that the tests regenerate (blah2_b200/scene.py):

  wh_long_<name>.npz   delayMin, delayMax, N, seed, ok (the reference's return value), seconds (its wall time on one
                       core), a, b, w (complex128, all nBins), and the filtered surveillance channel y' as a strided
                       subsample (every STEP-th sample), its norm and a seeded random projection of ALL samples (one
                       complex number that moves if any sample does), as oracle/gen_golden_full.py stores maps.

The reference solves by an O(nBins^3) Cholesky factorisation: minutes per case on one core.  Cases run in parallel
processes.

    python oracle/gen_golden_wh_long.py [name ...]
"""
import ctypes as C
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from blah2_b200.scene import make_scene  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
LIB = os.path.join(ROOT, "oracle", "_ref", "libblah2whlong.so")
STEP = 4099

# name: (delayMin, delayMax, N, seed); seed None = an all-zero reference channel (chol() fails at the first pivot)
CASES = {
    "t2049": (-10, 2039, 262144, 4101),      # first tap count above the one-sweep solve kernels
    "t2050": (-50, 2000, 2000000, 4102),     # blah2's default window at 10 MS/s
    "t2418": (0, 2418, 500000, 4103),        # last tap count whose old solve footprint (6 n double2) fits 227 KB
    "t2419": (5, 2424, 400000, 4104),        # the first that does not; delayMin > 0
    "t3585": (-20, 3565, 1000000, 4105),     # last tap count of the one-lag-block correlation plan
    "t3586": (0, 3586, 300000, 4106),        # first of the lag-block / partitioned plans
    "t4096": (-100, 3996, 1500000, 4107),    # the limit
    "t4096p": (7, 4103, 600000, 4108),       # the limit, delayMin > 0
    "fail4096": (-96, 4000, 300000, None),   # all-zero reference channel: the reference returns false
}


def projection(n, seed=7):
    """Unit-modulus pseudo-random weights over all samples (seeded; the tests rebuild them)."""
    rng = np.random.default_rng(seed)
    return np.exp(2j * np.pi * rng.random(n))


def case_inputs(delayMin, delayMax, n, seed):
    if seed is None:
        sc = make_scene(n, 2000000, seed=4100)
        return np.zeros(n, dtype=np.complex128), sc.y
    sc = make_scene(n, 2000000, seed=seed)
    return sc.x, sc.y


def run_reference(x, y, delayMin, delayMax):
    lib = C.CDLL(LIB, mode=os.RTLD_LOCAL)
    lib.refwh_process.restype = C.c_int
    lib.refwh_process.argtypes = [C.c_int32, C.c_int32, C.c_uint32] + [C.c_void_p] * 5
    nb = delayMax - delayMin
    x = np.ascontiguousarray(x, dtype=np.complex128)
    y = np.ascontiguousarray(y, dtype=np.complex128).copy()
    a, b, w = (np.zeros(nb, dtype=np.complex128) for _ in range(3))
    rc = lib.refwh_process(delayMin, delayMax, x.shape[0], x.ctypes.data, y.ctypes.data, a.ctypes.data, b.ctypes.data,
                           w.ctypes.data)
    assert rc in (0, 1), rc
    return bool(rc), y, a, b, w


def one(name):
    delayMin, delayMax, n, seed = CASES[name]
    x, y = case_inputs(delayMin, delayMax, n, seed)
    t0 = time.time()
    ok, yf, a, b, w = run_reference(x, y, delayMin, delayMax)
    sec = time.time() - t0
    np.savez_compressed(os.path.join(OUT, f"wh_long_{name}.npz"), delayMin=delayMin, delayMax=delayMax, N=n,
                        seed=-1 if seed is None else seed, ok=ok, seconds=sec, step=STEP, a=a, b=b, w=w,
                        sub=yf[::STEP].copy(), norm=float(np.linalg.norm(yf)), proj=np.sum(yf * projection(n)))
    return f"{name}: ok={ok} nBins={delayMax - delayMin} N={n} reference {sec:.1f} s"


def main():
    names = sys.argv[1:] or list(CASES)
    os.makedirs(OUT, exist_ok=True)
    with ProcessPoolExecutor(max_workers=min(len(names), os.cpu_count() or 1)) as ex:
        for line in ex.map(one, names):
            print(line, flush=True)


if __name__ == "__main__":
    main()
