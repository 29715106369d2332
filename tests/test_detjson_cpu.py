"""CPU: the detection document blah2 sends for every CPI, and the /stash/detection history its API serves.

b200dd_detjson_render_host (the product's formatter on the host) equals the compiled reference's documents stored in
tests/golden/detection_docs.npz and, where oracle/_ref/libblah2detjson.so was built, the reference live on a million
random detections.  oracle/stash_detection.py, the restatement of api/stash/detection.js that the GPU tests compare
the device history against, reproduces tests/golden/detection_stash.npz and hand-computed cases of its prune loop."""
import hashlib
import os

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import DetectionJson
from detjson_lists import LARGE, large_lists
from oracle import refdetjson
from oracle.stash_detection import Stash

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DOCS = np.load(os.path.join(GOLD, "detection_docs.npz"))
STASH = np.load(os.path.join(GOLD, "detection_stash.npz"))
SMALL = sorted(k[:-4] for k in DOCS.files if k.endswith("_doc"))


@pytest.mark.parametrize("name", SMALL)
def test_render_host_equals_the_stored_reference_documents(name):
    dl, dp, sn = DOCS[name + "_lists"]
    ts, fs = (int(v) for v in DOCS[name + "_meta"])
    assert DetectionJson.render_host(dl, dp, sn, ts, fs) == DOCS[name + "_doc"].tobytes()


@pytest.mark.parametrize("name", list(LARGE))
def test_render_host_equals_the_stored_reference_on_full_lists(name):
    doc = DetectionJson.render_host(*large_lists(name), LARGE[name]["ts"], LARGE[name]["fs"])
    assert len(doc) == int(DOCS[name + "_len"])
    assert hashlib.sha256(doc).digest() == DOCS[name + "_sha256"].tobytes()


@pytest.mark.skipif(not refdetjson.available(),
                    reason="compiled reference (oracle/_ref/libblah2detjson.so) not built")
def test_render_host_equals_the_live_reference_on_random_detections():
    rng = np.random.default_rng(7)
    total = 0
    while total < 1_000_000:
        n = int(rng.integers(1, 20000))
        # every magnitude the delay's km value stays finite for: random exponents, signs and significands
        v = []
        for _ in range(3):
            bits = rng.integers(0, 1 << 52, n, dtype=np.uint64) | (rng.integers(1023 - 60, 1023 + 90, n).astype(
                np.uint64) << np.uint64(52)) | (rng.integers(0, 2, n).astype(np.uint64) << np.uint64(63))
            v.append(bits.view(np.float64))
        fs = int(rng.choice([2000000, int(rng.integers(1, 1 << 32))]))
        ts = int(rng.integers(0, 1 << 63))
        assert DetectionJson.render_host(*v, ts, fs) == refdetjson.detection_json(*v, ts, fs), (fs, ts)
        total += n


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("where", [0, 1, 2])
def test_a_value_without_text_has_no_document(bad, where):
    v = [np.array([1.0, 2.0, 3.0]) for _ in range(3)]
    v[where][1] = bad
    with pytest.raises(capi.B200ddError) as e:
        DetectionJson.render_host(*v, 1, 2000000)
    assert e.value.code == capi.ERR_NONFINITE


def test_a_delay_whose_km_overflows_has_no_document():
    with pytest.raises(capi.B200ddError) as e:
        DetectionJson.render_host([1e308], [1.0], [1.0], 1, 1)
    assert e.value.code == capi.ERR_NONFINITE


@pytest.mark.parametrize("name", ["quirk", "above_2e53"])
def test_restatement_reproduces_the_stored_stash(name):
    docs, dlen = STASH[name + "_docs"].tobytes(), STASH[name + "_doc_len"]
    sent, slen = STASH[name + "_stash"].tobytes(), STASH[name + "_stash_len"]
    do, so = np.concatenate([[0], np.cumsum(dlen)]), np.concatenate([[0], np.cumsum(slen)])
    st = Stash()
    for i in range(dlen.size):
        if dlen[i]:
            st.push(docs[do[i]:do[i + 1]])
        assert st.send() == sent[so[i]:so[i + 1]], i


def _doc(ts, n=1, v=1.5):
    return DetectionJson.render_host([v] * n, [v] * n, [v] * n, ts, 2000000)


def test_stash_is_an_empty_array_before_the_first_document():
    st = Stash()
    assert st.send() == b"[]"
    st.push(b'{"timestamp":1,"delay":[1.0,')  # a truncated document changes nothing
    assert st.send() == b"[]"
    st.push(_doc(5, n=0))
    assert st.send() == b'{"timestamp":[],"delay":[],"doppler":[],"snr":[]}'


def test_prune_tests_every_other_document():
    st = Stash()
    for t in (0, 1000, 2000):  # three stale documents at the front ...
        st.push(_doc(t))
    st.push(_doc(302500))  # ... tests 0 (stale, shift), 2 (stale, shift), then i = 2 >= length 2: stop
    assert [m["timestamp"] for m in st.map] == [2000.0, 302500.0]
    assert st.send() == (b'{"timestamp":[2000,302500],"delay":[0.22,0.22],"doppler":[1.5,1.5],'
                         b'"snr":[1.5,1.5]}')


def test_zero_detection_documents_count_in_the_prune():
    st = Stash()
    st.push(_doc(0, n=2))
    st.push(_doc(10, n=0))  # holds a slot, sends nothing
    st.push(_doc(20, n=1))
    st.push(_doc(300021))  # tests 0 (stale: shift), then 20 at position 1 (stale: shift, the empty one goes), stop
    assert [m["timestamp"] for m in st.map] == [20.0, 300021.0]
    assert st.send() == b'{"timestamp":[20,300021],"delay":[0.22,0.22],"doppler":[1.5,1.5],"snr":[1.5,1.5]}'


def test_timestamps_above_2e53_are_numbers():
    st = Stash()
    st.push(_doc((1 << 53) + 1))
    st.push(_doc((1 << 53) + 3))
    assert st.send().startswith(b'{"timestamp":[9007199254740992,9007199254740996],')
    st.push(_doc(18446744073709551615))  # both are stale; the loop tests and removes only the first
    assert st.send().startswith(b'{"timestamp":[9007199254740996,18446744073709552000],')
