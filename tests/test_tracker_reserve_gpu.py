"""GPU: b200dd_tracker_reserve grows a live tracker without changing what it computes, and b200dd_tracker_usage reads
its live tracks and longest history.  A handle created at 16 tracks x 4 entries and grown before every CPI that
needs it renders, after every CPI, the documents of a handle created at the fixture's limits and of
tests/golden/track_docs.npz; refused and shrinking requests change nothing; an overflowed handle stays overflowed."""
import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import Tracker
from oracle.track_model import TrackModel
from track_sequences import load, matches, random_large_sequence, random_sequence, stored

pytestmark = pytest.mark.gpu
Z = load()
NAMES = [str(n) for n in Z["names"]]


def _fetch(tr, ts):
    try:
        return capi.OK, tr.fetch(ts)
    except capi.B200ddError as e:
        return e.code, b""


def _grow(tr, n_det, nh, cap, double):
    """Reserve by the rule for a CPI of n_det detections: exactly what it needs, or doubling."""
    live, longest = tr.usage()
    need = (live + n_det * nh, longest + 2)
    new = list(cap)
    for k in range(2):
        while new[k] < need[k]:
            new[k] = new[k] * 2 if double else need[k]
    if tuple(new) != tuple(cap):
        tr.reserve(*new)
    return tuple(new), tuple(new) != tuple(cap), live


def _run_grown(params, cpis, docs, double, big_limits=None):
    small = Tracker(*params, max_tracks=16, max_history=4, device=0)
    big = Tracker(*params, max_tracks=big_limits[0], max_history=big_limits[1], device=0) if big_limits else None
    mod = TrackModel(*params)
    nh = len(mod.acc_init)
    cap, grows, grows_past_1024 = (16, 4), [0, 0], 0
    for i, (d, f, s, ts) in enumerate(cpis):
        old = cap
        cap, grew, live = _grow(small, len(d), nh, cap, double)
        grows[0] += cap[0] > old[0]
        grows[1] += cap[1] > old[1]
        grows_past_1024 += grew and live > 1024
        small.process_host(d, f, s, ts)
        mod.process(d, f, ts)
        live, longest = small.usage()
        assert (live, longest) == (len(mod.tracks), max((len(t["hist"]) for t in mod.tracks), default=0)), i
        rc, doc = _fetch(small, ts)
        if big is not None:
            big.process_host(d, f, s, ts)
            assert _fetch(big, ts) == (rc, doc), i
        if docs is not None:
            want = docs[i]
            if want[3]:
                assert rc == capi.ERR_NONFINITE and doc == b"", i
            else:
                assert rc == capi.OK and matches(doc, want), (i, doc[:200])
        else:
            want = mod.to_json(ts, capi.format_track_doubles)
            assert (rc, doc) == ((capi.ERR_NONFINITE, b"") if want is None else (capi.OK, want)), i
    small.close()
    if big is not None:
        big.close()
    return grows, grows_past_1024


@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("name", NAMES)
def test_grown_handle_renders_the_stored_documents(name, double):
    params, limits, cpis, docs = stored(Z, name)
    grows, past = _run_grown(params, cpis, docs, double, big_limits=limits)
    if name == "large":
        assert grows[0] >= 2 and grows[1] >= 1 and past >= 1, (grows, past)


def test_grown_handle_on_random_sequences():
    rng = np.random.default_rng(404)
    for k in range(60):
        params, cpis = random_sequence(rng)
        _run_grown(params, cpis, None, double=bool(k % 2), big_limits=(4096, 128))


def test_grown_handle_with_thousands_of_tracks():
    rng = np.random.default_rng(1025)
    for k in range(2):
        params, cpis = random_large_sequence(rng)
        grows, past = _run_grown(params, cpis, None, double=bool(k % 2), big_limits=(1 << 16, 64))
        assert past >= 1 and grows[1] >= 1


def test_shrinking_and_refused_requests_change_nothing():
    params, limits, cpis, docs = stored(Z, "assoc")
    tr = Tracker(*params, max_tracks=limits[0], max_history=limits[1], device=0)
    lib = capi.load()
    half = len(cpis) // 2
    for d, f, s, ts in cpis[:half]:
        tr.process_host(d, f, s, ts)
    ts_half = cpis[half - 1][3]
    before, mb = tr.fetch(ts_half), tr.max_bytes
    tr.reserve(1, 1)  # raises neither limit
    tr.reserve(limits[0], limits[1])
    assert tr.max_bytes == mb and tr.fetch(ts_half) == before
    for t, h in [((1 << 24) + 1, 4), (16, (1 << 16) + 1), (1 << 24, 1 << 16)]:
        assert lib.b200dd_tracker_reserve(tr._h, t, h, None) == capi.ERR_ARG
        assert tr.max_bytes == mb and tr.fetch(ts_half) == before
    for i in range(half, len(cpis)):
        d, f, s, ts = cpis[i]
        tr.process_host(d, f, s, ts)
        assert matches(tr.fetch(ts), docs[i]), i
    tr.close()


def test_overflowed_handle_stays_overflowed():
    params, (max_tracks, max_hist), cpis, docs = stored(Z, "assoc")
    tr = Tracker(*params, max_tracks=max_tracks - 1, max_history=max_hist, device=0)
    over = None
    for i, (d, f, s, ts) in enumerate(cpis):
        if over is not None:
            tr.reserve(4 * max_tracks, 4 * max_hist)
        tr.process_host(d, f, s, ts)
        rc, doc = _fetch(tr, ts)
        if rc == capi.ERR_CAPACITY:
            over = i if over is None else over
        else:
            assert over is None and rc == capi.OK and matches(doc, docs[i]), i
    assert over is not None
    tr.reserve(4 * max_tracks, 4 * max_hist)
    assert _fetch(tr, cpis[-1][3]) == (capi.ERR_CAPACITY, b"")
    tr.reset()  # as new, at the grown limits
    for (d, f, s, ts), want in zip(cpis, docs):
        tr.process_host(d, f, s, ts)
        assert matches(tr.fetch(ts), want)
    tr.close()
