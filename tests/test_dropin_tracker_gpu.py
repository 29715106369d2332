"""GPU: the drop-in Tracker and Track classes against blah2's own, through the same class harness
(oracle/trackclass/track_class_capi.cpp) built with each: every sequence of tests/golden/track_docs.npz, random
sequences and the large sequence from the drop-in's first, small capacity give the same to_json text, get_n and
get_nState after every CPI; kept tracks are snapshots; save writes the same file; predict gives the same doubles.
An association at an unchanged timestamp is the documented difference: the drop-in's to_json returns ""."""
import numpy as np
import pytest

from oracle import track_class
from track_sequences import load, matches, random_large_sequence, random_sequence, stored

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not (track_class.available("ref") and track_class.available("dropin")),
                                 reason="class harnesses not built (build() with the blah2 sources)")]
Z = load()
NAMES = [str(n) for n in Z["names"]]
STATES = ("TENTATIVE", "ASSOCIATED", "ACTIVE", "COASTING", "active", "")


def _pair(params):
    return (track_class.TrackerClass("ref", *params[:5], fs=params[5], fc=params[6]),
            track_class.TrackerClass("dropin", *params[:5], fs=params[5], fc=params[6]))


def _compare(ref, dro, ts, k=-1, where=None):
    """The two tracks agree; returns the drop-in's document (b"" where a value is not finite)."""
    a, b = ref.to_json(ts, k), dro.to_json(ts, k)
    assert dro.get_n(k) == ref.get_n(k), where
    if b == b"":  # the reference's Writer stopped at a non-finite value
        assert a[:1] == b"{" and not a.endswith(b"]}"), where
        with pytest.raises(track_class.ClassError, match="non-finite"):
            dro.get_nState("ACTIVE", k)
        return b
    assert b == a, (where, b[:200], a[:200])
    for s in STATES:
        assert dro.get_nState(s, k) == ref.get_nState(s, k), (where, s)
    return b


def _run(params, cpis, docs=None):
    ref, dro = _pair(params)
    for i, (d, f, s, ts) in enumerate(cpis):
        ref.process(d, f, s, ts)
        dro.process(d, f, s, ts)
        doc = _compare(ref, dro, ts, where=i)
        if docs is not None:
            assert (doc == b"") == docs[i][3] and (doc == b"" or matches(doc, docs[i])), i
    ref.close()
    dro.close()


@pytest.mark.parametrize("name", NAMES)
def test_stored_sequences(name):
    params, _, cpis, docs = stored(Z, name)
    _run(params, cpis, docs)


def test_random_sequences():
    rng = np.random.default_rng(31)
    for _ in range(200):
        _run(*random_sequence(rng))


def test_thousands_of_tracks_from_the_first_capacity():
    params, _, cpis, docs = stored(Z, "large")
    _run(params, cpis, docs)
    rng = np.random.default_rng(64)
    _run(*random_large_sequence(rng))


def test_kept_tracks_are_snapshots():
    params, _, cpis, _ = stored(Z, "assoc")
    ref, dro = _pair(params)
    kept = []
    for i, (d, f, s, ts) in enumerate(cpis):
        ref.process(d, f, s, ts)
        dro.process(d, f, s, ts)
        if i % 4 == 1:
            kept.append((ref.keep(), dro.keep(), ts, dro.to_json(ts)))
    for kr, kd, ts, doc in kept:
        assert dro.to_json(ts, kd) == doc == ref.to_json(ts, kr)
        for other in (0, ts + 1, 2 ** 64 - 1):
            assert dro.to_json(other, kd) == ref.to_json(other, kr)
        assert dro.get_n(kd) == ref.get_n(kr)
        for s in STATES:
            assert dro.get_nState(s, kd) == ref.get_nState(s, kr)
    ref.close()
    dro.close()


def test_save_writes_the_same_file(tmp_path):
    params, _, cpis, _ = stored(Z, "config")
    ref, dro = _pair(params)
    for i, (d, f, s, ts) in enumerate(cpis):
        ref.process(d, f, s, ts)
        dro.process(d, f, s, ts)
        assert ref.save(ts, tmp_path / "ref.track") and dro.save(ts, tmp_path / "dropin.track")
    a, b = (tmp_path / "ref.track").read_bytes(), (tmp_path / "dropin.track").read_bytes()
    assert a == b and a.startswith(b'[{"timestamp":') and a.count(b'{"timestamp":') == len(cpis)
    for name, body in (("bad", b"{}"), ("open", b"[1,2")):
        for which, t in (("ref", ref), ("dropin", dro)):
            p = tmp_path / f"{name}.{which}"
            p.write_bytes(body)
            assert not t.save(0, p) and p.read_bytes() == body
    ref.close()
    dro.close()


def test_predict_is_bit_equal():
    rng = np.random.default_rng(9)
    for params in [(3, 5, 5, 1.0, 10.0, 2000000, 204640000), (2, 3, 4, 0.75, 3.0, 1234567, 98765432)]:
        ref, dro = _pair(params)
        for _ in range(2000):
            v = (rng.uniform(-500, 500), rng.uniform(-400, 400), rng.uniform(-50, 50), rng.uniform(0, 3))
            assert dro.predict(*v) == ref.predict(*v), v
        ref.close()
        dro.close()
    # TestTracker.cpp "Test predict": (10, -20) at 5 Hz/s over 1 s -> (9.821, -15) within 0.01
    dro = track_class.TrackerClass("dropin", 3, 5, 5, 1.0, 10.0, fs=2000000, fc=204640000)
    d, f = dro.predict(10, -20, 5, 1)
    assert abs(d - 9.821) < 0.01 and abs(f + 15) < 0.01
    dro.close()


def test_association_at_an_unchanged_timestamp():
    params = (1, 1, 1, 1.0, 2.0, 2000000, 204640000)  # m = n = 1: an association promotes
    cpis = [([0.5, 40.0], [0.3, 12.0], [20.0, 20.0], 5000),
            ([0.2, 80.0], [0.1, -30.0], [20.0, 20.0], 5000),  # T = 0: the association divides by zero
            ([60.0], [7.0], [20.0], 6000)] + [([], [], [], t) for t in (7000, 8000, 9000)] + \
           [([0.4, 90.0], [0.2, 3.0], [20.0, 20.0], 10000)]
    ref, dro = _pair(params)
    docs = []
    for d, f, s, ts in cpis:
        ref.process(d, f, s, ts)
        dro.process(d, f, s, ts)
        docs.append(_compare(ref, dro, ts))
    assert docs[1] == docs[2] == b"" and all(docs[k] for k in (0, 3, 4, 5, 6))  # the removals clear it
    ref.close()
    dro.close()
