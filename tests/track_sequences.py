"""Inputs of the tracker tests: the sequences stored in tests/golden/track_docs.npz, and random sequences shaped to
reach association, promotion, coasting, removals that skip tracks and id wrap-around quickly."""
from __future__ import annotations

import hashlib
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load():
    return np.load(os.path.join(GOLD, "track_docs.npz"))


def stored(z, name):
    """(params, limits, [(delay, doppler, snr, ts)], [(doc bytes or None, length, sha256, nonfinite)])"""
    p = f"{name}/"
    params = z[p + "params"]
    params = (int(params[0]), int(params[1]), int(params[2]), float(params[3]), float(params[4]), int(params[5]),
              int(params[6]))
    cnt = z[p + "count"]
    off = np.concatenate([[0], np.cumsum(cnt)])
    cpis = [tuple(z[p + k][off[i]:off[i + 1]] for k in ("delay", "doppler", "snr")) + (int(z[p + "ts"][i]),)
            for i in range(cnt.size)]
    docs, pos = [], 0
    raw = z[p + "docs"].tobytes()
    for i in range(cnt.size):
        n = int(z[p + "doc_len"][i])
        full = bool(z[p + "full"][i])
        docs.append((raw[pos:pos + n] if full else None, n, z[p + "sha256"][i].tobytes(), bool(z[p + "nonfinite"][i])))
        pos += n if full else 0
    return params, tuple(int(v) for v in z[p + "limits"]), cpis, docs


def matches(doc, want):
    """doc (bytes) equals the stored document `want` (from stored())."""
    full, n, sha, _ = want
    if full is not None:
        return doc == full
    return len(doc) == n and hashlib.sha256(doc).digest() == sha


def random_sequence(rng):
    """(params, [(delay, doppler, snr, ts)]) with small counts and frequent window hits."""
    m, n, nd = int(rng.integers(0, 5)), int(rng.integers(0, 7)), int(rng.integers(0, 6))
    cpi = float(rng.choice([0.3, 0.5, 0.75, 1.0]))
    params = (m, n, nd, cpi, float(rng.uniform(0, 6)), int(rng.choice([2000000, 3000000, 1234567])), 204640000)
    ts = 1731000000000
    cpis = []
    for _ in range(int(rng.integers(5, 30))):
        k = int(rng.integers(0, 5))
        d = rng.uniform(-3, 3, k) * (rng.random(k) < 0.6) + rng.uniform(-100, 100, k) * (rng.random(k) < 0.3)
        f = rng.uniform(-5, 5, k)
        ts += int(rng.choice([500, 750, 1000]))
        cpis.append((d, f, rng.uniform(10, 30, k), ts))
    return params, cpis


def random_large_sequence(rng, n_cpi=None):
    """(params, [(delay, doppler, snr, ts)]) with thousands of tracks at entry: 100-300 detections per CPI at a 1 s
    CPI (21 hypotheses each), nDelete 1-3, and CPIs with a detection in the association window (at a random place in
    the list) interleaved with CPIs without one, so the per-position counters differ and removals -- including
    removals that skip tracks -- fall on both sides of the update kernel's 1024-track chunks."""
    params = (1, int(rng.integers(1, 4)), int(rng.integers(1, 4)), 1.0, 10.0,  # m = 1: every association promotes
              int(rng.choice([2000000, 3000000, 1234567])), 204640000)
    ts = 1731000000000
    cpis = []
    for i in range(n_cpi or int(rng.integers(10, 15))):
        k = int(rng.integers(100, 300))
        d = rng.uniform(2, 400, k) * rng.choice([-1.0, 1.0], k)
        f = rng.uniform(-300, 300, k)
        if i % 3 == 1 or (i % 3 == 2 and rng.random() < 0.5):
            j = int(rng.integers(0, k))
            d[j], f[j] = rng.uniform(-0.9, 0.9), rng.uniform(-0.9, 0.9)
        ts += int(rng.choice([900, 1000, 1100]))
        cpis.append((d, f, rng.uniform(10, 30, k), ts))
    return params, cpis
