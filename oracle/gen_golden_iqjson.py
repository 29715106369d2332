"""Regenerate tests/golden/iqdata_docs.npz and tests/golden/iqdata_stash.npz.

TEST INFRASTRUCTURE ONLY.
  iqdata_docs.npz    spectra, metrics and timestamps with the compiled reference's own IqData::to_json(ts) of each
                     (oracle/refiqjson.py): small spectra stored with their documents (``_ok`` false where a bin has no
                     text and the stored text is the reference's truncated one); the 65536-bin spectrum of
                     tests/iqjson_spectra.py as length + SHA-256.
  iqdata_stash.npz   a timestamped document sequence longer than 20 and what /stash/iqdata serves after every document
                     (oracle/stash_iqdata.py, the restatement of api/stash/iqdata.js).  A document with a bin without
                     text is the reference's truncated text: JSON.parse rejects it and the stash does not change.

    python -m oracle.gen_golden_iqjson
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import refiqjson  # noqa: E402
from oracle.stash_iqdata import Stash  # noqa: E402
from iqjson_spectra import full_spectrum  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
OUT_DOCS = os.path.join(GOLD, "iqdata_docs.npz")
OUT_STASH = os.path.join(GOLD, "iqdata_stash.npz")
TS_MAX = 18446744073709551615


def _ulps(x, k=3):
    """x and its k neighbouring doubles on each side."""
    out = [x]
    lo = hi = x
    for _ in range(k):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        out += [lo, hi]
    return np.concatenate(out)


def special_bins():
    """(-0.01, 0) dB and (0, 0.01) dB; subnormal and 1e150-scale magnitudes."""
    near0 = np.array([0.9999, 0.99977, 0.999, 1 - 2 ** -40, 1.0, 1 + 2 ** -40, 1.001, 1.0023, 0.99770])
    return np.concatenate([near0, [5e-324, 1e-323j, 2.2250738585072014e-308, 1e-310 + 1e-310j, 1e150, 3e200 + 4e200j,
                                   1e-150j, 1.7976931348623157e308, 1e307 + 1e307j, -1e150, -3 - 4j]])


def boundary_bins():
    """Magnitudes whose 10 log10 lies within a few ulp of k/100, as real bins, as imaginary bins and split over both
    parts, then the special bins."""
    k = np.arange(-32000, 30001, 613)
    r = _ulps(10.0 ** (k / 1000.0))
    th = np.linspace(0.1, 1.4, r.size)
    return np.concatenate([r.astype(np.complex128), 1j * r, r * np.cos(th) + 1j * r * np.sin(th), special_bins()])


def doc_sets():
    """name -> (spectrum, (min, max, mean), timestamp)"""
    sets = {}
    sets["example"] = (np.array([1, 1e-3 + 2e-3j, 123 + 456j, 1e150]), (0.0, -1.005, 1e21), 1760000000123)
    sets["boundaries"] = (boundary_bins(), (-0.0, 1e21, -1.0), TS_MAX)
    sets["metrics_round"] = (np.array([2 + 1j, 0.5j]), (2.675, -0.005, 1.9999999999999998e21), 0)
    sets["metrics_small"] = (np.array([7 - 7j]), (0.009, -1e-300, 123456.789), (1 << 53) + 1)
    for c in "abcd":
        s = np.load(os.path.join(GOLD, f"spectrum_{c}.npz"))["spectrum"]
        sets[f"spectrum_{c}"] = (s, (0.0, 0.0, 0.0), 1731000000000 + ord(c))
    s = np.load(os.path.join(GOLD, "spectrum_a.npz"))["spectrum"]  # 2000 bins: blah2's bandwidth at config 2
    sets["zero_bin"] = (np.concatenate([s[:10], [0.0], s[10:20]]), (0.0, 0.0, 0.0), 1731000000100)
    sets["zero_first"] = (np.concatenate([[0j], s[:5]]), (0.0, 0.0, 0.0), 1731000000101)
    sets["nan_bin"] = (np.concatenate([s[:7], [complex(np.nan, 1.0)], s[7:9]]), (1.0, 2.0, 3.0), 1731000000102)
    sets["inf_bin"] = (np.concatenate([s[:3], [complex(0.0, np.inf)]]), (1.0, 2.0, 3.0), 1731000000103)
    return sets


def docs():
    out = {}
    for name, (s, m, ts) in doc_sets().items():
        doc = refiqjson.iqdata_json(s, *m, ts)
        ok = bool(np.all(np.isfinite(s)) and np.all(s != 0))
        out[f"{name}_spectrum"] = np.asarray(s, dtype=np.complex128)
        out[f"{name}_metrics"] = np.array(m, dtype=np.float64)
        out[f"{name}_ts"] = np.array(ts, dtype=np.uint64)
        out[f"{name}_ok"] = np.array(ok)
        out[f"{name}_doc"] = np.frombuffer(doc, dtype=np.uint8)
        print(f"{name}: {len(s)} bins, {len(doc)} bytes{'' if ok else ' (truncated)'}")
    doc = refiqjson.iqdata_json(full_spectrum(), 0.0, 0.0, 0.0, TS_MAX)
    out["full_len"] = np.array(len(doc), dtype=np.int64)
    out["full_sha256"] = np.frombuffer(hashlib.sha256(doc).digest(), dtype=np.uint8)
    print(f"full: {full_spectrum().size} bins, {len(doc)} bytes")
    return out


N_DOCS = 27
N_BINS = 64
BAD = {9: 0.0, 16: complex(np.nan, np.nan)}  # document -> the value one of its bins is set to


def sequence():
    """Timestamps and spectra of the stash sequence: the first 64 bins of spectrum_d scaled by a power of two per
    document, a few special bins, and two documents with a bin without text.  No bin sits within a few ulp of a 0.01
    boundary, where the device's log10 / hypot may differ from glibc's in the last bit, so the device's documents and
    stash can be compared with these byte for byte."""
    d = np.load(os.path.join(GOLD, "spectrum_d.npz"))["spectrum"][:N_BINS]
    extra = special_bins()
    ts = np.array([1731000000000 + 100 * i for i in range(N_DOCS)], dtype=np.uint64)
    ts[-1] = np.uint64(TS_MAX)
    ts[5] = ts[4]  # a repeated timestamp is taken as any other
    spectra = np.empty((N_DOCS, N_BINS), dtype=np.complex128)
    for i in range(N_DOCS):
        spectra[i] = d * np.ldexp(1.0, 3 * i - 40)
        spectra[i, 5:9] = extra[(4 * i) % (extra.size - 4):][:4]
        if i in BAD:
            spectra[i, 30] = BAD[i]
    return ts, spectra


METRICS = (-0.0, 1e21, 2.675)


def stash():
    ts, spectra = sequence()
    st = Stash()
    doc_bytes, doc_lens, sent_bytes, sent_lens = [], [], [], []
    for i in range(N_DOCS):
        doc = refiqjson.iqdata_json(spectra[i], *METRICS, int(ts[i]))
        st.push(doc)
        sent = st.send()
        doc_bytes.append(doc)
        doc_lens.append(len(doc))
        sent_bytes.append(sent)
        sent_lens.append(len(sent))
    print(f"stash: {N_DOCS} documents of {N_BINS} bins, last stash {sent_lens[-1]} bytes")
    return dict(ts=ts, spectra=spectra, metrics=np.array(METRICS), ok=np.array([i not in BAD for i in range(N_DOCS)]),
                doc_len=np.array(doc_lens, dtype=np.int64), docs=np.frombuffer(b"".join(doc_bytes), dtype=np.uint8),
                stash_len=np.array(sent_lens, dtype=np.int64),
                stash=np.frombuffer(b"".join(sent_bytes), dtype=np.uint8))


def main():
    assert refiqjson.available(), "build the oracle first (python __graft_entry__.py)"
    np.savez_compressed(OUT_DOCS, **docs())
    np.savez_compressed(OUT_STASH, **stash())
    for p in (OUT_DOCS, OUT_STASH):
        print(p, os.path.getsize(p), "bytes")


if __name__ == "__main__":
    main()
