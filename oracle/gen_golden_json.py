"""Regenerate tests/golden/map_json_*.npz from the compiled reference (oracle/_ref: libblah2json.so, libblah2ref.so).

TEST INFRASTRUCTURE ONLY.  The fixtures hold what blah2 sends on its map socket,
Map::delay_bin_to_km(Map::to_json(ts), fs) (src/data/Map.cpp:116-185), computed by the reference's own code
through oracle/json/ref_json_capi.cpp (set_metrics through oracle/ref_capi.cpp):
  map_json_values.npz  the text of single doubles (rapidjson Writer at 2 decimals, read back, written again):
                       every double within +-4 ulp of k/100 for |k| <= 100000 (as a code into candidate texts, see
                       tests/test_map_json_cpu.py), magnitudes below 0.01, +-0, and random bit patterns
  map_json_maps.npz    whole documents: small maps in full, config 2 / 3 / 5 sized maps as length + SHA-256, each
                       with the reference's set_metrics noisePower / maxPower.  The maps are generated from the cell
                       index by tests/map_json_maps.py, so only their parameters are stored.

    python -m oracle.gen_golden_json
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import refjson, refpath  # noqa: E402
from map_json_maps import MAPS, decimal_text, hash_map, k_grid  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


ref_texts = refjson.format_doubles
ref_document = refjson.map_json


def ref_metrics(m):
    lib = refpath.lib()
    lib.refpath_set_metrics.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    m = np.ascontiguousarray(m, dtype=np.complex128)
    met = np.zeros(2)
    lib.refpath_set_metrics(m.ctypes.data, m.shape[0], m.shape[1], met.ctypes.data)
    return float(met[0]), float(met[1])


def values_fixture(rng):
    ks, vals = k_grid()
    texts = ref_texts(vals.ravel())
    codes = np.full(vals.size, -1, dtype=np.int8)
    exc_idx, exc_txt = [], []
    for i, t in enumerate(texts):
        k = int(ks.ravel()[i])
        cand = (decimal_text(k - 1), decimal_text(k), decimal_text(k + 1), "0.0", "-0.0")
        if t in cand:
            codes[i] = cand.index(t)
        else:
            exc_idx.append(i)
            exc_txt.append(t)
    small = np.concatenate([
        np.array([0.0, -0.0, 0.01, -0.01, np.nextafter(0.01, 0), -np.nextafter(0.01, 0), 5e-324, -5e-324,
                  2.2250738585072014e-308, 0.00999999999999999, 0.009999999999999998]),
        rng.choice([-1.0, 1.0], 4096) * 10.0 ** rng.uniform(-323, -2, 4096),
    ])
    bits = rng.integers(0, 2 ** 64, 16384, dtype=np.uint64, endpoint=False)
    return dict(codes=codes.reshape(vals.shape), exc_idx=np.array(exc_idx, dtype=np.int64),
                exc_txt=np.frombuffer(",".join(exc_txt).encode(), dtype=np.uint8),
                small=small, small_txt=np.frombuffer(",".join(ref_texts(small)).encode(), dtype=np.uint8),
                bits=bits, bits_txt=np.frombuffer(",".join(ref_texts(bits.view(np.float64))).encode(), dtype=np.uint8))


def maps_fixture():
    out = {}
    for name, spec in MAPS.items():
        m, delay, doppler = hash_map(spec)
        noise, maxp = ref_metrics(m)
        doc = ref_document(m, delay, doppler, noise, maxp, spec["ts"], spec["fs"])
        out[f"{name}_metrics"] = np.array([noise, maxp])
        out[f"{name}_len"] = np.array(len(doc), dtype=np.int64)
        out[f"{name}_sha256"] = np.frombuffer(hashlib.sha256(doc).digest(), dtype=np.uint8)
        if spec.get("full"):
            out[f"{name}_doc"] = np.frombuffer(doc, dtype=np.uint8)
        print(f"{name}: {m.shape}, {len(doc)} bytes, noise {noise:.6f}, max {maxp:.6f}")
    return out


def main():
    assert refpath.available() and refjson.available(), "build the oracle first (python __graft_entry__.py)"
    rng = np.random.default_rng(20260115)
    np.savez_compressed(os.path.join(OUT, "map_json_values.npz"), **values_fixture(rng))
    np.savez_compressed(os.path.join(OUT, "map_json_maps.npz"), **maps_fixture())
    for f in ("map_json_values.npz", "map_json_maps.npz"):
        print(f, os.path.getsize(os.path.join(OUT, f)), "bytes")


if __name__ == "__main__":
    main()
