"""Regenerate tests/golden/detection_docs.npz and tests/golden/detection_stash.npz.

TEST INFRASTRUCTURE ONLY.
  detection_docs.npz   detection lists and the compiled reference's own
                       Detection::delay_bin_to_km(Detection::to_json(ts), fs) of each (oracle/refdetjson.py): small lists
                       stored with their documents; the 2^18-entry lists of tests/detjson_lists.py as length + SHA-256.
  detection_stash.npz  timestamped document sequences and what /stash/detection serves after every document
                       (oracle/stash_detection.py, the restatement of api/stash/detection.js).  A document whose
                       lists hold a non-finite value has no text (the reference's Writer stops): its length is 0 and
                       the stash does not change.

    python -m oracle.gen_golden_detjson
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import refdetjson  # noqa: E402
from oracle.stash_detection import Stash  # noqa: E402
from detjson_lists import LARGE, large_lists  # noqa: E402

OUT_DOCS = os.path.join(ROOT, "tests", "golden", "detection_docs.npz")
OUT_STASH = os.path.join(ROOT, "tests", "golden", "detection_stash.npz")
C = 299792458


def _near(x):
    """x and its two neighbouring doubles."""
    x = np.asarray(x, dtype=np.float64)
    return np.concatenate([np.nextafter(x, -np.inf), x, np.nextafter(x, np.inf)])


def small_sets():
    rng = np.random.default_rng(5)
    sets = {}
    sets["empty"] = (np.zeros(0), np.zeros(0), np.zeros(0), 0, 2000000)
    sets["one"] = (np.array([12.5]), np.array([-123.456]), np.array([17.3]), 1731000000000, 2000000)
    # x.xx5 boundaries and their neighbours, +-0.005, -0.0, |v| < 0.01; the delay bins land on the same km values
    k = np.arange(-3000, 3001, 7)
    b = np.concatenate([_near(k / 100 + 0.005), _near([0.005, -0.005, 0.0]), [-0.0, 0.004, -0.0099, 1e-300, 5e-324]])
    km_per_bin = C / 2000000 / 1000
    sets["boundaries"] = (b / km_per_bin, b, b[::-1].copy(), 1700000000123, 2000000)
    big = np.array([1e21, np.nextafter(1e21, 0), 1.5e22, -3e300, 1.7976931348623157e308, -1e21, 9.999999999999999e20])
    sets["huge"] = (np.array([1e21, -1e25, 1e300, 123.0, -5e20, 7e22, 0.5]), big, big[::-1].copy(), 18446744073709551615,
                    2000000)
    n = 40
    sets["negative_delay"] = (-rng.uniform(0, 60, n), rng.uniform(-500, 500, n), rng.uniform(5, 40, n), 1731000000002,
                              2000000)
    for fs in (1, 3, 999983, 2000001, 4294967295):
        n = 50
        sets[f"fs_{fs}"] = (rng.uniform(-100, 5000, n), rng.uniform(-2000, 2000, n), rng.uniform(-10, 60, n),
                            1731000000003, fs)
    z = np.load(os.path.join(ROOT, "tests", "golden", "full_cfg2.npz"))
    d = z["detections"]
    sets["cfg2_chain"] = (d[0], d[1], d[2], 1731000000004, int(z["geom"][4]))
    z = np.load(os.path.join(ROOT, "tests", "golden", "chain_a.npz"))
    d = z["interp"]
    sets["chain_a"] = (d[0], d[1], d[2], 1731000000005, int(z["geom"][4]))
    return sets


def docs():
    out = {}
    for name, (dl, dp, sn, ts, fs) in small_sets().items():
        doc = refdetjson.detection_json(dl, dp, sn, ts, fs)
        out[f"{name}_lists"] = np.stack([dl, dp, sn]).astype(np.float64)
        out[f"{name}_meta"] = np.array([ts, fs], dtype=np.uint64)
        out[f"{name}_doc"] = np.frombuffer(doc, dtype=np.uint8)
        print(f"{name}: {dl.size} detections, {len(doc)} bytes")
    for name, spec in LARGE.items():
        doc = refdetjson.detection_json(*large_lists(name), spec["ts"], spec["fs"])
        out[f"{name}_len"] = np.array(len(doc), dtype=np.int64)
        out[f"{name}_sha256"] = np.frombuffer(hashlib.sha256(doc).digest(), dtype=np.uint8)
        print(f"{name}: {len(doc)} bytes")
    return out


# name -> number of documents, first timestamp, seed
SEQS = {
    "quirk": dict(n=48, t0=1731000000000, seed=21),
    "above_2e53": dict(n=42, t0=(1 << 53) + 7, seed=22),
}


def sequence(spec):
    """Timestamps, detection counts and lists of one sequence: steps of 100 ms with bursts of stale documents
    (jumps beyond 300 s), irregular steps, zero-detection documents and one document with a NaN."""
    rng = np.random.default_rng(spec["seed"])
    n = spec["n"]
    steps = np.full(n, 100, dtype=np.int64)
    steps[0] = 0
    steps[10] = 300001  # the ten documents before are stale at once: every other one is tested
    steps[11:14] = 1
    steps[20] = 150000
    steps[21] = 150001
    steps[22:30] = rng.integers(1, 400000, 8)
    steps[35] = 900000
    steps[36:] = rng.integers(1, 200000, n - 36)
    ts = np.cumsum(steps).astype(np.uint64) + np.uint64(spec["t0"])
    counts = rng.integers(0, 7, n)
    counts[::7] = 0
    bad = np.zeros(n, dtype=bool)
    bad[23] = True
    counts[23] = max(counts[23], 1)
    total = int(counts.sum())
    lists = np.stack([rng.uniform(-5, 300, total), rng.uniform(-500, 500, total), rng.uniform(5, 40, total)])
    offs = np.concatenate([[0], np.cumsum(counts)])
    lists[2, offs[23]] = np.nan
    return ts, counts, lists, bad


def stash():
    out = {}
    for name, spec in SEQS.items():
        ts, counts, lists, bad = sequence(spec)
        total = int(counts.sum())
        offs = np.concatenate([[0], np.cumsum(counts)])
        st = Stash()
        doc_bytes, doc_lens, sent_bytes, sent_lens = [], [], [], []
        for i in range(ts.size):
            dl, dp, sn = (lists[k, offs[i]:offs[i + 1]] for k in range(3))
            if bad[i]:
                doc = b""
            else:
                doc = refdetjson.detection_json(dl, dp, sn, int(ts[i]), 2000000)
                st.push(doc)
            sent = st.send()
            doc_bytes.append(doc)
            doc_lens.append(len(doc))
            sent_bytes.append(sent)
            sent_lens.append(len(sent))
        out[f"{name}_ts"] = ts
        out[f"{name}_counts"] = counts.astype(np.int64)
        out[f"{name}_lists"] = lists
        out[f"{name}_doc_len"] = np.array(doc_lens, dtype=np.int64)
        out[f"{name}_docs"] = np.frombuffer(b"".join(doc_bytes), dtype=np.uint8)
        out[f"{name}_stash_len"] = np.array(sent_lens, dtype=np.int64)
        out[f"{name}_stash"] = np.frombuffer(b"".join(sent_bytes), dtype=np.uint8)
        print(f"{name}: {ts.size} documents, {total} detections, {len(st.map)} held at the end, last stash "
              f"{sent_lens[-1]} bytes")
    return out


def main():
    assert refdetjson.available(), "build the oracle first (python __graft_entry__.py)"
    np.savez_compressed(OUT_DOCS, **docs())
    np.savez_compressed(OUT_STASH, **stash())
    for p in (OUT_DOCS, OUT_STASH):
        print(p, os.path.getsize(p), "bytes")


if __name__ == "__main__":
    main()
