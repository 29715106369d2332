"""CPU: the map-JSON number formatter (blah2_b200/csrc/json_fmt.cuh, host path) gives rapidjson's text -- written
at two decimals, read back, written again, as Map::to_json + Map::delay_bin_to_km do -- for the stored value set
and, where the compiled reference exists, for fresh random doubles; map-JSON handles need a device."""
import ctypes as C
import os

import numpy as np
import pytest

from blah2_b200 import capi
from map_json_maps import decimal_text, k_grid

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "map_json_values.npz")


def _split(a):
    return a.tobytes().decode("ascii").split(",")


def expected_k_grid():
    z = np.load(GOLDEN)
    ks, vals = k_grid()
    codes = z["codes"].ravel()
    kk = ks.ravel()
    cand = {}
    out = []
    for i, c in enumerate(codes):
        k = int(kk[i])
        if c < 0:
            out.append(None)
            continue
        if k not in cand:
            cand[k] = (decimal_text(k - 1), decimal_text(k), decimal_text(k + 1), "0.0", "-0.0")
        out.append(cand[k][c])
    for i, t in zip(z["exc_idx"], _split(z["exc_txt"]) if z["exc_idx"].size else []):
        out[int(i)] = t
    assert all(t is not None for t in out)
    return vals.ravel(), out


def test_k_over_100_grid_matches_the_reference():
    vals, want = expected_k_grid()
    got = capi.format_doubles(vals)
    bad = [(float(vals[i]), got[i], want[i]) for i in range(len(want)) if got[i] != want[i]]
    assert not bad, bad[:10]
    # the values that make truncating the binary value wrong: the double nearest 12.34 lies below it
    assert capi.format_doubles([12.34, 1.102, 3.0, 0.005, -0.005, -0.0]) == ["12.34", "1.1", "3.0", "0.0", "-0.0",
                                                                              "-0.0"]


@pytest.mark.parametrize("key", ["small", "bits"])
def test_stored_values_match_the_reference(key):
    z = np.load(GOLDEN)
    vals = z[key] if key == "small" else z[key].view(np.float64)
    want = _split(z[key + "_txt"])
    got = capi.format_doubles(vals)
    assert len(got) == len(want) == vals.size
    bad = [(float(vals[i]), got[i], want[i]) for i in range(vals.size) if got[i] != want[i]]
    assert not bad, bad[:10]
    if key == "bits":  # NaN / inf patterns have no text
        assert sum(1 for t in want if t == "") == int(np.sum(~np.isfinite(vals)))


def test_random_doubles_match_the_live_reference():
    from oracle import refjson
    if not refjson.available():
        pytest.skip("the compiled reference (oracle/_ref) is not present")
    rng = np.random.default_rng(7)
    for chunk in range(10):
        bits = rng.integers(0, 2 ** 64, 10 ** 6, dtype=np.uint64)
        if chunk >= 5:  # half of them in the range of map values: dB around 0..800 in magnitude
            v = rng.uniform(-900.0, 900.0, 10 ** 6)
            bits = v.view(np.uint64)
        vals = bits.view(np.float64)
        want = refjson.format_doubles_bytes(vals)
        got = ",".join(capi.format_doubles(vals)).encode()
        if got != want:
            w, g = want.decode().split(","), got.decode().split(",")
            bad = [(vals[i], g[i], w[i]) for i in range(vals.size) if g[i] != w[i]]
            pytest.fail(f"{len(bad)} of {vals.size} differ: {bad[:5]}")


def test_format_doubles_reports_capacity():
    lib = capi.load()
    v = np.array([123.456, -7.0])
    out = np.empty(4, dtype=np.uint8)
    n = C.c_size_t()
    assert lib.b200dd_mapjson_format_doubles_host(capi.ptr(v), 2, capi.ptr(out), 4, C.byref(n)) == capi.ERR_CAPACITY
    assert n.value == len("123.45,-7.0")


def test_mapjson_needs_a_device():
    if capi.device_count() > 0:
        pytest.skip("a GPU is present")
    lib = capi.load()
    delay = np.arange(4, dtype=np.int32)
    doppler = np.arange(3, dtype=np.float64)
    h = C.c_void_p()
    assert lib.b200dd_mapjson_create(3, 4, capi.ptr(delay), capi.ptr(doppler), 2000000, -1, C.byref(h)) == capi.ERR_CUDA
    assert lib.b200dd_mapjson_create(0, 4, capi.ptr(delay), capi.ptr(doppler), 2000000, -1, C.byref(h)) == capi.ERR_ARG
    assert lib.b200dd_mapjson_create(3, 4, None, capi.ptr(doppler), 2000000, -1, C.byref(h)) == capi.ERR_ARG
