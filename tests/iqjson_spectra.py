"""The 65536-bin spectrum of the IQ-data JSON tests (the C ABI's bound), built from tests/golden/spectrum_c.npz by
exact operations only (scaling by powers of two, conjugation), so every machine builds the same bits.  Shared by
oracle/gen_golden_iqjson.py, which stores its document as length + SHA-256, and the tests."""
import os

import numpy as np

N_FULL = 65536
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def full_spectrum() -> np.ndarray:
    c = np.load(os.path.join(GOLD, "spectrum_c.npz"))["spectrum"]
    j = np.arange(N_FULL)
    rep = j // c.size
    s = c[j % c.size] * np.ldexp(1.0, rep * 7 - 56)
    return np.where(rep % 2 == 1, np.conj(s), s)
