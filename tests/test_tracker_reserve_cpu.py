"""CPU: the capacity rule the drop-in Tracker reserves by before every CPI -- live + n (2 nAcc + 1) tracks and
longest + 2 history entries for n detections -- holds the tracks after the CPI, on the CPU model of the tracker, over
random sequences and the fixture's large sequence; the reserve / usage entry points refuse null handles; and the
drop-in Tracker refuses a rangeRes or lambda that is not c / f of an integer f."""
import ctypes as C

import numpy as np
import pytest

from blah2_b200 import capi
from oracle import track_class
from oracle.track_model import TrackModel
from track_sequences import load, random_sequence, stored


def _check_rule(params, cpis):
    mod = TrackModel(*params)
    nh = len(mod.acc_init)
    for i, (d, f, s, ts) in enumerate(cpis):
        live = len(mod.tracks)
        longest = max((len(t["hist"]) for t in mod.tracks), default=0)
        want_tracks, want_hist = live + len(d) * nh, longest + 2
        mod.process(d, f, ts)
        after = max((len(t["hist"]) for t in mod.tracks), default=0)
        assert len(mod.tracks) <= want_tracks and after <= want_hist, (i, len(mod.tracks), want_tracks, after)
    return len(mod.tracks)


def test_rule_on_random_sequences():
    rng = np.random.default_rng(2024)
    for _ in range(2000):
        _check_rule(*random_sequence(rng))


def test_rule_on_the_large_sequence():
    params, _, cpis, _ = stored(load(), "large")
    assert _check_rule(params, cpis) > 16000


def test_reserve_and_usage_refuse_null():
    lib = capi.load()
    a, b = C.c_uint32(), C.c_uint32()
    assert lib.b200dd_tracker_reserve(None, 16, 4, None) == capi.ERR_ARG
    assert lib.b200dd_tracker_usage(None, C.byref(a), C.byref(b), None) == capi.ERR_ARG


@pytest.mark.skipif(not track_class.available("dropin"), reason="drop-in class harness not built")
@pytest.mark.parametrize("range_res, lam", [(1.5, 299792458 / 204640000), (299792458 / 2000000, 1e-9),
                                            (-149.896229, 1.0), (float("nan"), 1.0), (0.0, 1.0)])
def test_dropin_constructor_refuses_non_integer_rates(range_res, lam):
    with pytest.raises(track_class.ClassError, match="rangeRes|lambda"):
        track_class.TrackerClass("dropin", 3, 5, 5, 1.0, 10.0, range_res=range_res, lam=lam)
