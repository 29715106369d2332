"""Regenerate tests/golden/track_docs.npz.

TEST INFRASTRUCTURE ONLY.  For each sequence: the tracker parameters, the detection list and timestamp of every CPI,
and the compiled reference's own tracker->process(detection, ts)->to_json(ts) after every CPI
(oracle/reftracker.py): full bytes for small documents, length + SHA-256 for large ones.  A CPI whose document holds
a non-finite value is flagged: the reference's Writer stops there and its text is truncated.  `limits` holds the
most live tracks and the longest history the sequence reaches (the CPU model, oracle/track_model.py, counts them).

    python -m oracle.gen_golden_tracker
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.reftracker import RefTracker  # noqa: E402
from oracle.track_model import TrackModel  # noqa: E402
from track_sequences import random_large_sequence  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "track_docs.npz")
FULL_MAX = 1 << 16  # documents up to this size are stored whole
FC = 204640000
T0 = 1731000000000


def _near_zero(rng, k):
    """k detections, about half inside the association window of a 0.75 s CPI."""
    inside = rng.random(k) < 0.5
    d = np.where(inside, rng.uniform(-0.99, 0.99, k), rng.uniform(-40, 80, k))
    f = np.where(inside, rng.uniform(-1.3, 1.3, k), rng.uniform(-300, 300, k))
    return d, f, rng.uniform(10, 30, k)


def sequences():
    rng = np.random.default_rng(2024)
    seqs = {}

    def add(name, params, cpis):
        seqs[name] = (params, cpis)

    # association, promotion and COASTING: most CPIs hold a detection in the window
    add("assoc", (2, 3, 4, 0.75, 3.0, 2000000, FC),
        [(*_near_zero(rng, int(rng.integers(0, 4))), T0 + 750 * i) for i in range(24)])
    # the config's values (M 3, N 5, delete 10, maxAcc 10) at a 1 s CPI: 21 hypotheses per detection
    add("config", (3, 5, 10, 1.0, 10.0, 2000000, FC),
        [(*_near_zero(rng, int(rng.integers(1, 4))), T0 + 1000 * i) for i in range(16)])
    # removals that skip tracks: nothing associates, nDelete 2
    cp = []
    for i in range(14):
        k = int(rng.integers(0, 8))
        cp.append((rng.uniform(5, 60, k), rng.uniform(-200, 200, k), rng.uniform(10, 20, k), T0 + 500 * i))
    add("skips", (3, 5, 2, 0.5, 10.0, 3000000, FC), cp)
    # nDelete = 0: every reached track is removed
    add("ndelete0", (1, 2, 0, 0.75, 3.0, 2000000, FC),
        [(*_near_zero(rng, int(rng.integers(0, 3))), T0 + 750 * i) for i in range(12)])
    # empty lists between non-empty ones, and m = n = 0
    cp = []
    for i in range(12):
        k = 0 if i % 3 else int(rng.integers(1, 3))
        cp.append((*_near_zero(rng, k), T0 + 750 * i))
    add("empty", (0, 0, 3, 0.75, 3.0, 2000000, FC), cp)
    # values of 1e21 and more, negative values: tentative first, then associated and sent
    big_d = np.array([1e22, -3.5e21, 123456.789, -0.004])
    big_f = np.array([-5e21, 2.5e23, -777.77, 1e21])
    cp = [(big_d, big_f, np.zeros(4), T0)]
    cp += [(np.array([0.25]), np.array([-0.5]), np.zeros(1), T0 + 750 * (i + 1)) for i in range(4)]
    add("exponent", (1, 1, 5, 0.75, 1.0, 2000000, FC), cp)
    # T = 0: an association with the same timestamp makes an infinite / NaN acceleration
    cp = [(np.array([0.5, 30.0]), np.array([0.2, 40.0]), np.zeros(2), T0),
          (np.array([0.1]), np.array([0.3]), np.zeros(1), T0),
          (np.array([0.2]), np.array([0.1]), np.zeros(1), T0 + 750),
          (np.array([]), np.array([]), np.zeros(0), T0 + 1500)]
    add("t0", (1, 1, 5, 0.75, 1.0, 2000000, FC), cp)
    # id wrap: 3200 detections x 21 hypotheses = 67200 adds (past FFFE), then one association sends them all
    k = 3200
    cp = [(rng.uniform(2, 60, k), rng.uniform(-400, 400, k), np.zeros(k), T0),
          (np.array([0.5]), np.array([0.25]), np.zeros(1), T0 + 1000),
          (rng.uniform(2, 60, 5), rng.uniform(-400, 400, 5), np.zeros(5), T0 + 2000)]
    add("idwrap", (1, 1, 1000, 1.0, 10.0, 2000000, FC), cp)
    # the Interpolate lists of the committed chain fixtures, perturbed over 16 CPIs, three in four with a detection
    # in the window
    za = np.load(os.path.join(ROOT, "tests", "golden", "chain_a.npz"))
    zb = np.load(os.path.join(ROOT, "tests", "golden", "full_cfg2.npz"))
    lists = [za["interp"], zb["detections"]]
    g = za["geom"]
    cp = []
    for i in range(16):
        d, f, s = (np.array(v, dtype=np.float64) for v in lists[i % 2])
        d = d + 0.25 * i
        f = f - 1.5 * i
        if i % 4 != 3:
            d, f, s = np.append(d, 0.125 * (i % 5) - 0.3), np.append(f, 0.05 * i - 0.4), np.append(s, 12.0)
        cp.append((d, f, s, T0 + 500 * i))
    add("chain", (3, 5, 10, float(g[5]) / float(g[4]), 10.0, int(g[4]), FC), cp)
    # thousands of tracks at entry with removals that skip tracks on both sides of the update kernel's 1024-track
    # chunks (tests/track_sequences.py), from its own generator so that the sequences above stay as they were
    add("large", *random_large_sequence(np.random.default_rng(1024), n_cpi=14))
    return seqs


def main():
    arrays = {}
    names = []
    for name, (params, cpis) in sequences().items():
        names.append(name)
        ref = RefTracker(*params)
        mod = TrackModel(*params)
        docs, lens, shas, nonfinite = [], [], [], []
        most_tracks = most_hist = 1
        for d, f, s, ts in cpis:
            doc = ref.process(d, f, s, ts)
            mod.process(d, f, ts)
            most_tracks = max(most_tracks, len(mod.tracks))
            most_hist = max([most_hist] + [len(t["hist"]) for t in mod.tracks])
            try:
                json.loads(doc)
                nonfinite.append(0)
            except ValueError:
                nonfinite.append(1)
            lens.append(len(doc))
            shas.append(np.frombuffer(hashlib.sha256(doc).digest(), dtype=np.uint8))
            docs.append(doc if len(doc) <= FULL_MAX else b"")
        ref.close()
        p = f"{name}/"
        arrays[p + "params"] = np.array(params, dtype=np.float64)
        arrays[p + "limits"] = np.array([most_tracks, most_hist], dtype=np.int64)
        arrays[p + "count"] = np.array([len(c[0]) for c in cpis], dtype=np.int64)
        for k, key in enumerate(("delay", "doppler", "snr")):
            arrays[p + key] = np.concatenate([np.asarray(c[k], dtype=np.float64) for c in cpis])
        arrays[p + "ts"] = np.array([c[3] for c in cpis], dtype=np.uint64)
        arrays[p + "doc_len"] = np.array(lens, dtype=np.int64)
        arrays[p + "sha256"] = np.stack(shas)
        arrays[p + "full"] = np.array([len(x) > 0 for x in docs], dtype=bool)
        arrays[p + "docs"] = np.frombuffer(b"".join(docs), dtype=np.uint8)
        arrays[p + "nonfinite"] = np.array(nonfinite, dtype=bool)
        print(f"{name}: {len(cpis)} CPIs, tracks <= {most_tracks}, history <= {most_hist}, "
              f"docs {min(lens)}..{max(lens)} B, {sum(nonfinite)} non-finite")
    arrays["names"] = np.array(names)
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
