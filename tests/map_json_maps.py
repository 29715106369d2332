"""Inputs of the map-JSON fixtures (tests/golden/map_json_*.npz), generated instead of stored.

Maps come from the cell index through splitmix64 in unsigned 64-bit integer arithmetic, and every float step is
exact (24-bit integers times powers of two in float32), so they do not depend on the numpy version or platform.
"""
from __future__ import annotations

import numpy as np

# name -> shape, seed, fs, timestamp; "full": the fixture stores the whole document, else length + SHA-256.
# cfg2 / cfg3 / cfg5 have the map sizes of BASELINE configs 2, 3 and 5.
MAPS = {
    "tiny": dict(nDop=3, nDel=4, seed=1, fs=2000000, ts=1700000000123, delay0=-2, full=True),
    "small": dict(nDop=17, nDel=33, seed=2, fs=10000000, ts=18446744073709551615, delay0=0, full=True),
    "medium": dict(nDop=64, nDel=40, seed=3, fs=20000000, ts=0, delay0=-5, full=True),
    "cfg2": dict(nDop=257, nDel=300, seed=4, fs=2000000, ts=1731000000000, delay0=0),
    "cfg3": dict(nDop=1025, nDel=512, seed=5, fs=10000000, ts=1731000000001, delay0=0),
    "cfg5": dict(nDop=4097, nDel=512, seed=6, fs=20000000, ts=1731000000002, delay0=0),
}


def splitmix64(x):
    x = x + np.uint64(0x9E3779B97F4A7C15)
    z = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def hash_map(spec):
    """(map complex128 [nDop, nDel] holding float32 values, delay int32 [nDel], doppler float64 [nDop])."""
    nDop, nDel = spec["nDop"], spec["nDel"]
    n = nDop * nDel
    with np.errstate(over="ignore"):
        h = splitmix64(np.arange(n, dtype=np.uint64) + np.uint64(spec["seed"] << 40))
    re = ((h >> np.uint64(40)).astype(np.int64) - (1 << 23)).astype(np.float32)
    im = (((h >> np.uint64(16)) & np.uint64(0xFFFFFF)).astype(np.int64) - (1 << 23)).astype(np.float32)
    # magnitudes over 2^-8 .. 2^7 times a 24-bit integer: tens of dB of spread like a real map
    scale = np.exp2((h & np.uint64(15)).astype(np.int32) - 8).astype(np.float32)
    re, im = re * scale, im * scale
    peaks = (np.arange(n) % 997) == 5  # strong targets, 2^16 above their neighbours
    re[peaks] *= np.float32(65536.0)
    im[peaks] *= np.float32(65536.0)
    both0 = (re == 0) & (im == 0)
    re[both0] = np.float32(1.0)  # |z| = 0 has no JSON text
    # cells near the float32 extremes
    ext = [(3.0e38, 1.0e38), (1.0e-45, 0.0), (-1.17549435e-38, 2.0e-40), (0.0, -3.4028235e38), (-1.4e-45, -1.4e-45)]
    for i, (a, b) in enumerate(ext):
        j = (7 + 131 * i) % n
        re[j], im[j] = np.float32(a), np.float32(b)
    m = (re.astype(np.float64) + 1j * im.astype(np.float64)).reshape(nDop, nDel)
    delay = (np.arange(nDel) + spec["delay0"]).astype(np.int32)
    doppler = (np.arange(nDop, dtype=np.float64) - nDop // 2) * (spec["fs"] / (nDop * 4096.0 + 13.0))
    return m, delay, doppler


def k_grid():
    """(k [200001, 9], values [200001, 9]): the doubles within +-4 ulp of k/100, |k| <= 100000."""
    k = np.arange(-100000, 100001, dtype=np.int64)
    base = k / 100.0
    cols = [base]
    up, dn = base.copy(), base.copy()
    for _ in range(4):
        up = np.nextafter(up, np.inf)
        dn = np.nextafter(dn, -np.inf)
        cols.append(up)
        cols.insert(0, dn)
    vals = np.stack(cols, axis=1)
    return np.repeat(k[:, None], 9, axis=1), vals


def decimal_text(k: int) -> str:
    """rapidjson's two-decimal text of the decimal k/100: "12.34", "12.3", "12.0", "-0.05"."""
    s = "-" if k < 0 else ""
    ip, fp = divmod(abs(k), 100)
    frac = ("%02d" % fp).rstrip("0") or "0"
    return f"{s}{ip}.{frac}"
