"""CPU: the tracker's parallel form (oracle/track_model.py) is blah2's Tracker + Track::to_json, document for document:
against every document stored in tests/golden/track_docs.npz, and against the compiled reference
(oracle/_ref/libblah2tracker.so) on random sequences where it was built.  b200dd_tracker_plan's hypothesis count
and parameter checks."""
import json

import numpy as np
import pytest

from blah2_b200 import capi
from oracle import reftracker
from oracle.track_model import TrackModel, hypotheses
from track_sequences import load, matches, random_large_sequence, random_sequence, stored

Z = load()
NAMES = [str(n) for n in Z["names"]]


@pytest.mark.parametrize("name", NAMES)
def test_model_matches_stored_documents(name):
    params, limits, cpis, docs = stored(Z, name)
    mod = TrackModel(*params)
    most_tracks = most_hist = 1
    for i, ((d, f, s, ts), want) in enumerate(zip(cpis, docs)):
        mod.process(d, f, ts)
        most_tracks = max(most_tracks, len(mod.tracks))
        most_hist = max([most_hist] + [len(t["hist"]) for t in mod.tracks])
        doc = mod.to_json(ts, capi.format_track_doubles)
        if want[3]:  # the reference's Writer stopped at a non-finite value
            assert doc is None, (name, i)
        else:
            assert doc is not None and matches(doc, want), (name, i)
    assert (most_tracks, most_hist) == limits


def _iterations(mod, delay, doppler, n_delete):
    """D and which iterations run, for the CPI mod is about to process (the parallel form, oracle/track_model.py)."""
    n0 = len(mod.tracks)
    assoc = any(-1.0 < d < 1.0 and mod.dop_lo < f < mod.dop_hi for d, f in zip(delay, doppler))
    D = np.array([(0 if assoc else mod._c(i)) + 1 > n_delete for i in range(n0)], dtype=bool)
    r = np.concatenate([[0], np.cumsum(D)[:-1]]).astype(np.int64)
    run = np.arange(n0) + r < n0
    return D, r, run


def test_fixture_covers_the_quirks():
    """The stored sequences reach what the parallel form has to get right, including removals past the update
    kernel's first 1024-track chunk, where the removal count carried from earlier chunks is non-zero."""
    seen = dict(coasting=False, wrap=False, nonfinite=False, exponent=False, skip=False, skip_past_chunk=False,
                carry_past_chunk=False, process_past_chunk=False)
    for name in NAMES:
        params, _, cpis, docs = stored(Z, name)
        mod = TrackModel(*params)
        for (d, f, s, ts), want in zip(cpis, docs):
            D, r, run = _iterations(mod, d, f, params[2])
            mod.process(d, f, ts)
            seen["nonfinite"] |= want[3]
            if want[0] is not None and not want[3]:
                doc = json.loads(want[0])
                seen["coasting"] |= doc["nCoasting"] > 0
                seen["exponent"] |= b"e2" in want[0]
            ids = [t["id"] for t in mod.tracks]  # new tracks take increasing ids until the counter wraps
            seen["wrap"] |= any(v < u for u, v in zip(ids, ids[1:]))
            # a removal that skips a track: two removals in a row among the iterations that ran
            rem = D & run
            pairs = np.nonzero(rem[:-1] & rem[1:])[0]
            seen["skip"] |= pairs.size > 0
            seen["skip_past_chunk"] |= bool((pairs >= 1024).any())
            past = np.nonzero(rem)[0]
            seen["carry_past_chunk"] |= bool(((past >= 1024) & (r[past] > 0)).any())
            seen["process_past_chunk"] |= bool((run & (np.arange(run.size) % 1024 + r >= 1024)).any())
    assert all(seen.values()), seen


@pytest.mark.skipif(not reftracker.available(), reason="oracle/_ref/libblah2tracker.so not built")
def test_model_matches_live_reference():
    rng = np.random.default_rng(20241016)
    n_docs = n_nonfinite = 0
    for _ in range(2000):
        params, cpis = random_sequence(rng)
        ref = reftracker.RefTracker(*params)
        mod = TrackModel(*params)
        for d, f, s, ts in cpis:
            want = ref.process(d, f, s, ts)
            mod.process(d, f, ts)
            doc = mod.to_json(ts, capi.format_track_doubles)
            if doc is None:
                n_nonfinite += 1
                with pytest.raises(ValueError):
                    json.loads(want)
            else:
                assert doc == want
            n_docs += 1
        ref.close()
    assert n_docs > 20000


@pytest.mark.skipif(not reftracker.available(), reason="oracle/_ref/libblah2tracker.so not built")
def test_model_matches_live_reference_with_thousands_of_tracks():
    rng = np.random.default_rng(4096)
    most = 0
    for _ in range(3):
        params, cpis = random_large_sequence(rng)
        ref = reftracker.RefTracker(*params)
        mod = TrackModel(*params)
        for d, f, s, ts in cpis:
            most = max(most, len(mod.tracks))
            want = ref.process(d, f, s, ts)
            mod.process(d, f, ts)
            assert mod.to_json(ts, capi.format_track_doubles) == want
        ref.close()
    assert most > 4096


def _params(**kw):
    p = dict(m=3, n=5, nDelete=10, cpi=0.75, maxAcc=10.0, fs=2000000, fc=204640000)
    p.update(kw)
    return p


def test_plan_hypotheses():
    for cpi, acc, nh in [(0.75, 10.0, 11), (1.0, 10.0, 21), (0.5, 10.0, 5), (0.5, 3.9, 1), (0.1, 10.0, 1),
                         (1.0, 4096.0, 8193), (0.75, -0.5, 1), (0.0, 10.0, 1)]:
        assert capi.tracker_plan(**_params(cpi=cpi, maxAcc=acc))[0] == nh, (cpi, acc)
        assert len(hypotheses(cpi, acc)) == nh


def test_plan_bounds():
    nh, mb, db = capi.tracker_plan(**_params(), max_tracks=1000, max_history=64)
    assert db == 1000 * (16 * 64 + 4 * 4 + 52)
    assert mb > 1000 * 64 * 63
    capi.tracker_plan(**_params(), max_tracks=1 << 16, max_history=512)


@pytest.mark.parametrize("kw", [dict(maxAcc=float("nan")), dict(maxAcc=3e9), dict(maxAcc=-3e9),
                                dict(cpi=100.0), dict(cpi=float("nan")), dict(cpi=float("inf")),
                                dict(maxAcc=-2.0, cpi=1.0), dict(maxAcc=4097.0, cpi=1.0), dict(fs=0), dict(fc=0),
                                dict(max_tracks=0), dict(max_tracks=(1 << 24) + 1), dict(max_history=0),
                                dict(max_history=(1 << 16) + 1), dict(max_tracks=1 << 16, max_history=1 << 12)])
def test_plan_rejects(kw):
    lim = dict(max_tracks=kw.pop("max_tracks", 1024), max_history=kw.pop("max_history", 64))
    with pytest.raises(capi.B200ddError) as e:
        capi.tracker_plan(**_params(**kw), **lim)
    assert e.value.code == capi.ERR_ARG
    if "cpi" in kw or "maxAcc" in kw:
        p = _params(**kw)
        h = hypotheses(p["cpi"], p["maxAcc"])
        assert h is None or len(h) > 8193
