"""CPU: the host render of the timing document is the reference's Timing::to_json, byte for byte (the stored documents
of tests/golden/timing_docs.npz, and the compiled reference live where it was built); the restatement of
api/stash/timing.js gives the stored /stash/timing bytes after every document; the C ABI refuses bad arguments."""
import ctypes as C
import os

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import timing_render_host
from oracle import reftiming
from oracle.stash_timing import N_CPI, Stash

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DOCS = np.load(os.path.join(GOLD, "timing_docs.npz"))
STASH = np.load(os.path.join(GOLD, "timing_stash.npz"))
STAGES = ["extract_buffer", "spectrum", "clutter_filter", "ambiguity_processing", "detector", "tracker",
          "output_radar_data", "cpi"]


def _cases():
    names = DOCS["names"].tobytes().decode().split("\n")
    vo = np.concatenate([[0], np.cumsum(DOCS["count"])])
    do = np.concatenate([[0], np.cumsum(DOCS["doc_len"])])
    docs = DOCS["docs"].tobytes()
    for i in range(DOCS["doc_len"].size):
        nm = names[i].split(",") if DOCS["count"][i] else []
        yield (int(DOCS["t_start"][i]), int(DOCS["t_now"][i]), int(DOCS["n"][i]), nm, DOCS["values"][vo[i]:vo[i + 1]],
               docs[do[i]:do[i + 1]])


def test_host_render_equals_the_stored_reference_documents():
    n = 0
    for t0, t, k, names, v, doc in _cases():
        assert timing_render_host(t0, t, k, names, v) == doc, doc
        n += 1
    assert n == DOCS["doc_len"].size > 60


def test_the_stored_documents_reach_the_cases_that_matter():
    docs = [c[-1].decode() for c in _cases()]
    assert any('"uptime_s":18446744073709552.0' in d for d in docs)  # the wrapped uptime
    assert any(d.startswith('{"timestamp":9007199254740992,') for d in docs)
    assert any(d.startswith('{"timestamp":18446744073709551615,"nCpi":18446744073709551615,') for d in docs)
    assert any('"uptime_days":248.0,' in d for d in docs)
    assert any('1e21' in d for d in docs) and any('1.5e22' in d for d in docs)
    body = ",".join(docs)
    assert body.count('":0.0,') > 3 and '":0.01,' in body and '":0.1,' in body
    # the neighbours of 0.01 (k = 2) print on both sides of the boundary of the truncated text
    assert '"extract_buffer":0.0,"spectrum":0.0,"clutter_filter":0.01,' in body or '":0.0,"' in body
    assert len({c[-1] for c in _cases()}) == len(docs)
    keysets = {tuple(k for k in STAGES if f'"{k}":' in d) for d in docs}
    assert len(keysets) >= 16


def test_restatement_gives_the_stored_stash_after_every_document():
    dlen, slen = STASH["doc_len"], STASH["stash_len"]
    docs, sent = STASH["docs"].tobytes(), STASH["stash"].tobytes()
    do, so = np.concatenate([[0], np.cumsum(dlen)]), np.concatenate([[0], np.cumsum(slen)])
    assert dlen.size == 27
    st = Stash()
    assert st.send() == STASH["empty"].tobytes() == b"{}"
    for i in range(dlen.size):
        st.push(docs[do[i]:do[i + 1]])
        assert st.send() == sent[so[i]:so[i + 1]], i
    last = sent[so[-2]:so[-1]].decode()
    assert last.startswith('{"timestamp":[') and '"nCpi"' not in last
    assert last.index('"cpi"') < last.index('"tracker"')  # first-seen order
    assert len(st.output["timestamp"]) == N_CPI and len(st.output["tracker"]) == N_CPI - 1


def test_restatement_ignores_a_document_it_cannot_parse():
    st = Stash()
    st.push(b'{"timestamp":5,"nCpi":1,"uptime_s":0.0,"uptime_days":0.0,"cpi":1.5}')
    before = st.send()
    assert before == b'{"timestamp":[5],"uptime_s":[0],"uptime_days":[0],"cpi":[1.5]}'
    st.push(b'{"timestamp":6,"nCpi":2,"uptime_s":0.0,')
    assert st.send() == before


def test_bad_arguments_are_refused():
    lib = capi.load()
    out = np.empty(4096, dtype=np.uint8)
    n = C.c_size_t(7)
    names = (C.c_char_p * 2)(b"cpi", b"x")
    v = np.array([1.0, 2.0])
    assert lib.b200dd_timing_render_host(0, 0, 0, names, capi.ptr(v), 2, None, 4096, C.byref(n)) == capi.ERR_ARG
    assert n.value == 0
    assert lib.b200dd_timing_render_host(0, 0, 0, None, capi.ptr(v), 2, capi.ptr(out), 4096, None) == capi.ERR_ARG
    assert lib.b200dd_timing_render_host(0, 0, 0, names, None, 2, capi.ptr(out), 4096, None) == capi.ERR_ARG
    assert lib.b200dd_timing_render_host(0, 0, 0, None, None, 0, capi.ptr(out), 4096, None) == capi.OK
    assert lib.b200dd_timing_render_host(0, 0, 0, (C.c_char_p * 2)(b"cpi", None), capi.ptr(v), 2, capi.ptr(out),
                                         4096, None) == capi.ERR_ARG
    big = np.zeros(17)
    assert lib.b200dd_timing_render_host(0, 0, 0, (C.c_char_p * 17)(*[b"a"] * 17), capi.ptr(big), 17, capi.ptr(out),
                                         4096, None) == capi.ERR_ARG
    for bad in (b'a"b', b"a\\b", b"a\nb", b"\xc3\xa9", b"x" * 64):
        with pytest.raises(capi.B200ddError) as e:
            timing_render_host(0, 0, 0, [bad], [1.0])
        assert e.value.code == capi.ERR_ARG
    assert timing_render_host(0, 0, 0, [b"x" * 63], [1.0]).endswith(b'"' + b"x" * 63 + b'":1.0}')
    for bad in (np.nan, np.inf, -np.inf):
        with pytest.raises(capi.B200ddError) as e:
            timing_render_host(0, 0, 0, ["cpi"], [bad])
        assert e.value.code == capi.ERR_ARG
    doc = timing_render_host(0, 0, 0, ["cpi"], [1.0])
    assert lib.b200dd_timing_render_host(0, 0, 0, names, capi.ptr(v), 1, capi.ptr(out), len(doc) - 1,
                                         C.byref(n)) == capi.ERR_CAPACITY
    assert n.value == len(doc)
    assert lib.b200dd_timing_max_bytes() >= 13 + 20 + 8 + 20 + 16 * 90
    # the pipeline entry points refuse a null handle or output without a device
    cnt = C.c_uint32()
    assert lib.b200dd_pipeline_enable_timing_json(None, 0, None, None) == capi.ERR_ARG
    assert lib.b200dd_pipeline_fetch_timing_json(None, 0, capi.ptr(out), 4096, C.byref(n)) == capi.ERR_ARG
    assert lib.b200dd_pipeline_fetch_timing_stash(None, capi.ptr(out), 4096, C.byref(n)) == capi.ERR_ARG
    assert lib.b200dd_pipeline_debug_timing_values(None, None, None, 0, C.byref(cnt)) == capi.ERR_ARG


def test_python_binding_declares_the_timing_entry_points():
    declared = {name for name, _, _ in capi.SIGNATURES}
    assert {"b200dd_timing_render_host", "b200dd_timing_max_bytes", "b200dd_pipeline_enable_timing_json",
            "b200dd_pipeline_fetch_timing_json", "b200dd_pipeline_fetch_timing_stash",
            "b200dd_pipeline_debug_timing_values"} <= declared
    from blah2_b200.process import Pipeline
    for m in ("enable_timing_json", "fetch_timing_json", "fetch_timing_stash", "timing_values"):
        assert callable(getattr(Pipeline, m))


@pytest.mark.skipif(not reftiming.available(), reason="the compiled reference is built where the blah2 sources exist")
def test_host_render_equals_the_live_reference_on_random_value_sets():
    rng = np.random.default_rng(31)
    for i in range(100000):
        mask = rng.integers(0, 2, len(STAGES)).astype(bool)
        names = [s for s, m in zip(STAGES, mask) if m]
        scale = 10.0 ** rng.uniform(-4, 6 if i % 100 else 24)
        v = rng.uniform(0, 1, len(names)) * scale
        if i % 7 == 0:  # next to a 0.005 boundary
            v = np.round(v * 200) / 200 + rng.integers(-3, 4, len(names)) * np.spacing(v)
        t0 = int(rng.integers(0, 1 << 64, dtype=np.uint64)) if i % 11 == 0 else 1731000000000
        t = int(rng.integers(0, 1 << 64, dtype=np.uint64)) if i % 13 == 0 else t0 + int(rng.integers(0, 1 << 40))
        t &= (1 << 64) - 1
        k = int(rng.integers(1, 1 << 63))
        assert timing_render_host(t0, t, k, names, v) == reftiming.timing_json(t0, t, k, names, v), (t0, t, k, v)
