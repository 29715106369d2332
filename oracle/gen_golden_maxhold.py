"""Regenerate tests/golden/maxhold_docs.npz: what /stash/map serves after every CPI of the sequences of
tests/maxhold_maps.py.

TEST INFRASTRUCTURE ONLY.  Each CPI's map document is the compiled reference's own
Map::delay_bin_to_km(Map::to_json(ts), fs) (oracle/refjson.py), with the reference's set_metrics values
(oracle/refpath.py).  oracle/stash_maxhold.py, the restatement of api/stash/maxhold.js, turns the documents into the
bytes the API sends.  The zero-cell CPI has no document (rapidjson cannot write the cell), so the stash never sees
it.  Stored per sequence: the metrics of every CPI, and the documents in full (tiny, small, medium) or as length +
SHA-256 (config 2, 3 and 5 sizes); a length of 0 marks a CPI with no document.

    python -m oracle.gen_golden_maxhold
"""
from __future__ import annotations

import hashlib
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import refjson, refpath  # noqa: E402
from oracle.gen_golden_json import ref_metrics  # noqa: E402
from oracle.stash_maxhold import Stash  # noqa: E402
from maxhold_maps import N_SEQ, SEQS, seq_map, timestamp  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "maxhold_docs.npz")


def sequence(name, spec):
    stash = Stash()
    metrics, lens, shas, docs = [], [], [], []
    t0 = time.time()
    for i in range(N_SEQ):
        noise, maxp = ref_metrics(seq_map(spec, i, with_zero=False)[0])
        metrics.append((noise, maxp))
        if spec.get("zero_cpi") == i:
            lens.append(0)
            shas.append(bytes(32))
            continue
        m, delay, doppler = seq_map(spec, i)
        stash.push(refjson.map_json(m, delay, doppler, noise, maxp, timestamp(spec, i), spec["fs"]))
        sent = stash.send()
        lens.append(len(sent))
        shas.append(hashlib.sha256(sent).digest())
        docs.append(sent)
    out = {f"{name}_metrics": np.array(metrics), f"{name}_len": np.array(lens, dtype=np.int64),
           f"{name}_sha256": np.frombuffer(b"".join(shas), dtype=np.uint8).reshape(N_SEQ, 32)}
    if spec.get("full"):
        out[f"{name}_docs"] = np.frombuffer(b"".join(docs), dtype=np.uint8)
    print(f"{name}: {N_SEQ} CPIs, last document {lens[-1]} bytes, {time.time() - t0:.1f} s")
    return out


def main():
    assert refpath.available() and refjson.available(), "build the oracle first (python __graft_entry__.py)"
    out = {}
    for name, spec in SEQS.items():
        out.update(sequence(name, spec))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
