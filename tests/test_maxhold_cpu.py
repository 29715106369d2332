"""CPU: the max-hold cell text (blah2_b200/csrc/json_fmt.cuh jf::hundredths + jf::fmt_hundredths, host path) is
what blah2's API sends at /stash/map for a cell: the map document's text parsed by JSON.parse and re-printed by
Number::toString (oracle/stash_maxhold.py js_number_text); max-hold handles need a device."""
import ctypes as C
import os

import numpy as np
import pytest

from blah2_b200 import capi
from oracle.stash_maxhold import Stash, js_number_text

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "map_json_values.npz")
INT32_HUNDREDTHS = 2 ** 31 / 100  # a cell text at or beyond this has no int32 hundredths


# ECMA-262 Number::toString results, as a JS engine prints them
JS_TABLE = [
    (0.0, "0"), (-0.0, "0"), (12.0, "12"), (-12.5, "-12.5"), (0.1 + 0.2, "0.30000000000000004"), (1e21, "1e+21"),
    (1e-7, "1e-7"), (1e-6, "0.000001"), (123e-20, "1.23e-18"), (float(2 ** 64 - 1), "18446744073709552000"),
    (float(2 ** 53 + 1), "9007199254740992"), (5e-324, "5e-324"), (1.7976931348623157e308, "1.7976931348623157e+308"),
    (123456789012345680000.0, "123456789012345680000"), (1.5e22, "1.5e+22"), (0.01, "0.01"), (-0.29, "-0.29"),
    (100.0, "100"), (21474836.47, "21474836.47"),
]


@pytest.mark.parametrize("v,text", JS_TABLE)
def test_js_number_text_table(v, text):
    assert js_number_text(v) == text


def _check(vals, texts, got):
    """got[i] == Number::toString(JSON.parse(texts[i])) where the cell has int32 hundredths, "" elsewhere."""
    assert len(got) == len(texts) == len(vals)
    uniq = {t: (js_number_text(float(t)) if t and abs(float(t)) < INT32_HUNDREDTHS else "") for t in set(texts)}
    bad = [(float(vals[i]), t, got[i], uniq[t]) for i, t in enumerate(texts) if got[i] != uniq[t]]
    assert not bad, bad[:10]


@pytest.mark.parametrize("key", ["k_grid", "small", "bits"])
def test_cell_text_of_every_stored_value(key):
    """The stored reference texts of map_json_values.npz: the k/100 +- 4 ulp grid, the small values, the bit
    patterns.  An empty field exactly where the stored text is empty or out of int32 range."""
    from test_map_json_cpu import expected_k_grid
    z = np.load(GOLDEN)
    if key == "k_grid":
        vals, texts = expected_k_grid()
    else:
        vals = z[key] if key == "small" else z[key].view(np.float64)
        texts = z[key + "_txt"].tobytes().decode("ascii").split(",")
    got = capi.format_maxhold_doubles(vals)
    _check(vals, texts, got)
    if key == "bits":
        assert sum(1 for t in got if t == "") >= int(np.sum(~np.isfinite(vals)))


def test_cell_text_of_random_doubles():
    rng = np.random.default_rng(17)
    for chunk in range(10):
        if chunk < 5:
            vals = rng.integers(0, 2 ** 64, 10 ** 6, dtype=np.uint64).view(np.float64)
        else:  # map values: dB around 0..800 in magnitude, and values near the int32 edge
            vals = rng.uniform(-900.0, 900.0, 10 ** 6) if chunk < 9 else rng.uniform(-2.2e7, 2.2e7, 10 ** 6)
        _check(vals, capi.format_doubles(vals), capi.format_maxhold_doubles(vals))


def test_stash_restatement():
    """Window of 20, the latest header, per-cell max, JSON.stringify's number texts."""
    st = Stash()
    def doc(ts, noise, cells):
        return (b'{"timestamp":%d,"nRows":1,"nCols":2,"noisePower":%s,"maxPower":3.0,"delay":[-0.15,0.0],'
                b'"doppler":[0.0],"data":[[%s]]}' % (ts, noise, cells))
    st.push(doc(2 ** 64 - 1, b"1.5", b"-0.0,7.25"))
    assert st.send() == (b'{"timestamp":18446744073709552000,"nRows":1,"nCols":2,"noisePower":1.5,"maxPower":3,'
                         b'"delay":[-0.15,0],"doppler":[0],"data":[[0,7.25]]}')
    for i in range(20):
        st.push(doc(i, b"2.0", b"%d.0,-1.0" % -i))
    assert st.send().endswith(b'"noisePower":2,"maxPower":3,"delay":[-0.15,0],"doppler":[0],"data":[[0,-1]]}')
    st.push(doc(21, b"2.0", b"-30.0,-5.0"))  # the window now holds CPIs -1 .. -19 and this one
    assert st.send().endswith(b'"data":[[-1,-1]]}')


def test_format_maxhold_doubles_reports_capacity():
    lib = capi.load()
    v = np.array([123.456, -7.0])
    out = np.empty(4, dtype=np.uint8)
    n = C.c_size_t()
    assert lib.b200dd_maxhold_format_doubles_host(capi.ptr(v), 2, capi.ptr(out), 4, C.byref(n)) == capi.ERR_CAPACITY
    assert n.value == len("123.45,-7")


def test_maxhold_needs_a_device():
    if capi.device_count() > 0:
        pytest.skip("a GPU is present")
    from blah2_b200.process import MaxHold
    with pytest.raises(capi.B200ddError) as e:
        MaxHold(np.arange(4, dtype=np.int32), np.arange(3, dtype=np.float64), 2000000)
    assert e.value.code == capi.ERR_CUDA
    lib = capi.load()
    h = C.c_void_p()
    delay, doppler = np.arange(4, dtype=np.int32), np.arange(3, dtype=np.float64)
    assert lib.b200dd_maxhold_create(0, 4, capi.ptr(delay), capi.ptr(doppler), 2000000, -1, C.byref(h)) == capi.ERR_ARG
    assert lib.b200dd_maxhold_create(3, 4, None, capi.ptr(doppler), 2000000, -1, C.byref(h)) == capi.ERR_ARG
