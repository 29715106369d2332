"""Inputs of the detection-JSON fixtures (tests/golden/detection_docs.npz, detection_stash.npz).

The small lists are stored in the fixture; the 2^18-entry lists come from the entry index through splitmix64 in
unsigned 64-bit integer arithmetic, assembled bit by bit into doubles, so they do not depend on the numpy version
or platform.
"""
from __future__ import annotations

import numpy as np

from map_json_maps import splitmix64

N_FULL = 1 << 18  # the detection lists' capacity

# name -> seed, fs, timestamp and the exponent range of the values (|v| in [2^lo, 2^hi)); "bounded" lists keep
# every value's hundredths inside int32, so the stash can hold them
LARGE = {
    "random_full": dict(seed=11, fs=2000000, ts=1731000000000, lo=-40, hi=90),
    "bounded_full": dict(seed=12, fs=3000017, ts=1731000000001, lo=-10, hi=23),
}


def hash_doubles(n, seed, lo, hi):
    """n doubles with random signs, random 52-bit significands and exponents uniform in [lo, hi)."""
    with np.errstate(over="ignore"):
        h = splitmix64(np.arange(n, dtype=np.uint64) + np.uint64(seed << 40))
    e = (h & np.uint64(0x7FF)) % np.uint64(hi - lo)
    sign = (h >> np.uint64(11)) & np.uint64(1)
    bits = (sign << np.uint64(63)) | ((e + np.uint64(1023 + lo)) << np.uint64(52)) | (h >> np.uint64(12))
    return bits.view(np.float64)


def large_lists(name):
    """(delay bins, doppler, snr) of a LARGE entry."""
    s = LARGE[name]
    return tuple(hash_doubles(N_FULL, 3 * s["seed"] + k, s["lo"], s["hi"]) for k in range(3))
