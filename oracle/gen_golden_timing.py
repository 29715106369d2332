"""Writes tests/golden/timing_docs.npz and tests/golden/timing_stash.npz from the compiled reference
(oracle/_ref/libblah2timing.so: Timing::update + Timing::to_json) and the restatement of api/stash/timing.js
(oracle/stash_timing.py).  TEST INFRASTRUCTURE ONLY.

timing_docs.npz, one case per document: t_start, t_now, n (uint64), the stage names (one line per case, comma
separated) and their values (float64, flattened, `count` per case), and the reference's bytes (`docs`, `doc_len`).
The cases cover values a few ulp either side of 0.005 boundaries, 0, values under 0.005, large values (an exponent
form included), uptimes past 248 days, a wrapped uptime, timestamps of 2^53 and more, and every combination of the
optional stages (spectrum, clutter_filter, detector, tracker).

timing_stash.npz: a 27-document sequence (`docs`, `doc_len`) and the /stash/timing bytes after each (`stash`,
`stash_len`), plus the bytes before the first (`empty`).  The tracker's key appears mid-sequence, so first-seen order
puts it last.

    python -m oracle.gen_golden_timing
"""
from __future__ import annotations

import itertools
import os

import numpy as np

from oracle import reftiming
from oracle.stash_timing import Stash

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
T0 = 1731000000000


def stage_names(spectrum, clutter, detector, tracker):
    """blah2's keys in blah2's order (blah2.cpp:251-338) for one stage combination."""
    return (["extract_buffer"] + (["spectrum"] if spectrum else []) + (["clutter_filter"] if clutter else [])
            + ["ambiguity_processing"] + (["detector"] if detector else []) + (["tracker"] if tracker else [])
            + ["output_radar_data", "cpi"])


def boundary_values():
    """Doubles a few ulp either side of k * 0.005, plus 0 and values under 0.005."""
    out = [0.0, 1e-300, 5e-324, 0.001, 0.0049999999999999, 0.004999999999999999]
    for k in list(range(1, 40)) + [199, 200, 201, 2001, 20001, 200001, 2000001]:
        c = k * 0.005
        for u in range(-3, 4):
            v = c
            for _ in range(abs(u)):
                v = np.nextafter(v, np.inf if u > 0 else -np.inf)
            out.append(float(v))
    return out


def doc_cases(rng):
    cases = []
    combos = list(itertools.product((False, True), repeat=4))
    for i, c in enumerate(combos):
        names = stage_names(*c)
        cases.append((T0, T0 + 100 * i, i + 1, names, rng.uniform(0, 5, len(names))))
    b = boundary_values()
    names = stage_names(True, True, True, True)
    for j in range(0, len(b), len(names)):
        v = (b[j:j + len(names)] + [0.0] * len(names))[:len(names)]
        cases.append((T0, T0 + 7 * j, 30 + j, names, np.array(v)))
    for v in (1e3, 123456.789, 1e15, 9.99e20, 1e21, 1.5e22, 1.7976931348623157e308):
        cases.append((T0, T0 + 1, 2, names[:2], np.array([v, v / 3])))
    day = 86400000
    for up in (248 * day, 248 * day + 1, 2 ** 31, 2 ** 32 + 5, 10 ** 15, 2 ** 53 + 1):
        cases.append((T0, T0 + up, 7, names, rng.uniform(0, 50, len(names))))
    cases.append((T0, T0 - 1, 3, names, rng.uniform(0, 50, len(names))))  # wrapped uptime
    cases.append((0, 0, 0, [], np.zeros(0)))
    for ts in (2 ** 53, 2 ** 53 + 1, 10 ** 15, 10 ** 15 + 1, 2 ** 64 - 1):
        cases.append((T0, ts, 2 ** 64 - 1, names, rng.uniform(0, 50, len(names))))
    return cases


def pack(cases):
    docs = [reftiming.timing_json(*c) for c in cases]
    return dict(
        t_start=np.array([c[0] for c in cases], dtype=np.uint64),
        t_now=np.array([c[1] for c in cases], dtype=np.uint64),
        n=np.array([c[2] for c in cases], dtype=np.uint64),
        count=np.array([len(c[3]) for c in cases], dtype=np.int32),
        names=np.frombuffer("\n".join(",".join(c[3]) for c in cases).encode(), dtype=np.uint8),
        values=np.concatenate([np.asarray(c[4], dtype=np.float64) for c in cases]),
        docs=np.frombuffer(b"".join(docs), dtype=np.uint8),
        doc_len=np.array([len(d) for d in docs], dtype=np.int64),
    )


def stash_sequence(rng):
    """27 documents of one pipeline run: the tracker is enabled from the 9th on."""
    cases = []
    for i in range(27):
        names = stage_names(True, True, True, i >= 8)
        v = rng.uniform(0, 3, len(names))
        v[-1] = v[:-1].sum()
        cases.append((T0 - 5000, T0 + 250 * i, i + 1, names, v))
    return cases


def main():
    rng = np.random.default_rng(53)
    np.savez_compressed(os.path.join(GOLD, "timing_docs.npz"), **pack(doc_cases(rng)))
    seq = pack(stash_sequence(rng))
    st = Stash()
    empty = st.send()
    sent, do = [], np.concatenate([[0], np.cumsum(seq["doc_len"])])
    docs = seq["docs"].tobytes()
    for i in range(seq["doc_len"].size):
        st.push(docs[do[i]:do[i + 1]])
        sent.append(st.send())
    np.savez_compressed(os.path.join(GOLD, "timing_stash.npz"), docs=seq["docs"], doc_len=seq["doc_len"],
                        stash=np.frombuffer(b"".join(sent), dtype=np.uint8),
                        stash_len=np.array([len(s) for s in sent], dtype=np.int64),
                        empty=np.frombuffer(empty, dtype=np.uint8))


if __name__ == "__main__":
    main()
