"""CPU: the host render of the IQ-data document is the reference's IqData::to_json, byte for byte (the stored
documents of tests/golden/iqdata_docs.npz, and the compiled reference live where it was built), and the restatement
of api/stash/iqdata.js gives the stored /stash/iqdata bytes after every document."""
import hashlib
import os

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import IqDataJson
from iqjson_spectra import N_FULL, full_spectrum
from oracle import refiqjson
from oracle.stash_iqdata import N_CPI, Stash

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DOCS = np.load(os.path.join(GOLD, "iqdata_docs.npz"))
STASH = np.load(os.path.join(GOLD, "iqdata_stash.npz"))
NAMES = sorted(k[:-4] for k in DOCS.files if k.endswith("_doc"))


def _case(name):
    return (DOCS[name + "_spectrum"], tuple(DOCS[name + "_metrics"]), int(DOCS[name + "_ts"]),
            DOCS[name + "_doc"].tobytes(), bool(DOCS[name + "_ok"]))


@pytest.mark.parametrize("name", NAMES)
def test_host_render_equals_the_stored_reference_documents(name):
    s, m, ts, doc, ok = _case(name)
    if ok:
        assert IqDataJson.render_host(s, *m, ts) == doc
        return
    # the reference's Writer stops at the first bin without text, after that bin's separator
    with pytest.raises(capi.B200ddError) as e:
        IqDataJson.render_host(s, *m, ts)
    assert e.value.code == capi.ERR_NONFINITE
    k = int(np.flatnonzero(~np.isfinite(s) | (s == 0))[0])
    prefix = IqDataJson.render_host(s[:k], *m, ts)
    assert doc == prefix[:-2] + (b"," if k else b"")


def test_host_render_of_the_full_spectrum():
    s = full_spectrum()
    assert s.size == N_FULL
    doc = IqDataJson.render_host(s, 0.0, 0.0, 0.0, 18446744073709551615)
    assert len(doc) == int(DOCS["full_len"])
    assert hashlib.sha256(doc).digest() == DOCS["full_sha256"].tobytes()


def test_the_stored_documents_reach_the_cases_that_matter():
    doc = DOCS["boundaries_doc"].tobytes().decode()
    body = doc[doc.index('"spectrum":[') + 12:-2].split(",")
    assert doc.startswith('{"timestamp":18446744073709551615,"min":-0.0,"max":1e21,"mean":-1.0,"frequency":[],')
    assert "-0.0" in body and "0.0" in body
    assert min(float(v) for v in body) < -3200 and max(float(v) for v in body) > 3000  # subnormal, near DBL_MAX
    # the 7 neighbouring magnitudes around each 10^(k/1000) straddle a 0.01 boundary for some k
    s = DOCS["boundaries_spectrum"]
    groups = (s.size - 9 - 11) // 3
    real = np.array(body[:groups]).reshape(7, -1)
    assert sum(len(set(real[:, j])) > 1 for j in range(real.shape[1])) >= 5
    assert DOCS["metrics_round_doc"].tobytes().startswith(b'{"timestamp":0,"min":2.67,"max":-0.0,"mean":1.9999999999999997e21,')


def test_non_finite_metrics_are_rejected():
    for m in ((np.nan, 0.0, 0.0), (0.0, np.inf, 0.0), (0.0, 0.0, -np.inf)):
        with pytest.raises(capi.B200ddError) as e:
            IqDataJson.render_host([1.0], *m, 1)
        assert e.value.code == capi.ERR_ARG


def test_restatement_gives_the_stored_stash_after_every_document():
    dlen, slen = STASH["doc_len"], STASH["stash_len"]
    docs, sent = STASH["docs"].tobytes(), STASH["stash"].tobytes()
    do, so = np.concatenate([[0], np.cumsum(dlen)]), np.concatenate([[0], np.cumsum(slen)])
    assert dlen.size > N_CPI + 5
    st = Stash()
    assert st.send() == b"[]"
    for i in range(dlen.size):
        st.push(docs[do[i]:do[i + 1]])
        assert st.send() == sent[so[i]:so[i + 1]], i
    assert len(st.spectrum) == N_CPI
    assert sent[so[-2]:so[-1]].startswith(b'{"timestamp":[')
    assert b'],"min":0,"max":1e+21,"mean":2.67,"frequency":[[],[],' in sent[so[-2]:so[-1]]
    assert sent[so[-2]:so[-1]].count(b"[]") == N_CPI


def test_restatement_keeps_the_stash_on_a_truncated_document():
    st = Stash()
    st.push(b'{"timestamp":5,"min":0.0,"max":0.0,"mean":0.0,"frequency":[],"spectrum":[1.5,-0.0]}')
    before = st.send()
    assert before == b'{"timestamp":[5],"min":0,"max":0,"mean":0,"frequency":[[]],"spectrum":[[1.5,0]]}'
    st.push(b'{"timestamp":6,"min":0.0,"max":0.0,"mean":0.0,"frequency":[],"spectrum":[1.5,')
    assert st.send() == before


@pytest.mark.skipif(not refiqjson.available(), reason="the compiled reference is built where the blah2 sources exist")
def test_host_render_equals_the_live_reference_on_random_spectra():
    rng = np.random.default_rng(29)
    for _ in range(300):
        n = int(rng.integers(1, 2500))
        s = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 10.0 ** rng.uniform(-320, 305, n)
        s[s == 0] = 1.0
        m = rng.standard_normal(3) * 10.0 ** rng.uniform(-4, 24, 3)
        ts = int(rng.integers(0, 1 << 64, dtype=np.uint64))
        assert IqDataJson.render_host(s, *m, ts) == refiqjson.iqdata_json(s, *m, ts)
