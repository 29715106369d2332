"""Time blah2's Tracker / Track classes per CPI -- tracker.process(&detection, ts) then track->to_json(ts), as
blah2.cpp:291-296 and :324-328 run them -- with the reference's own classes on one host core and with the drop-in
classes on the device, through the same class harness (oracle/_ref/libtrackclass_{ref,dropin}.so), on the loads of
tools/time_tracker.py.  The drop-in's time includes its capacity check and the growth of its tracker.

    python tools/time_dropin_tracker.py [--cpis 36] [--warmup 24] [--ref-max-adds 6000]

The reference is timed only where ndet x hypotheses (the tracks each CPI adds) is at most --ref-max-adds.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from blah2_b200 import capi  # noqa: E402
from oracle import track_class  # noqa: E402
from time_tracker import FS, FC, sequence  # noqa: E402


def run(which, ndet, cpi, n_cpi, warmup):
    seq = sequence(ndet, n_cpi, cpi, seed=ndet)
    tr = track_class.TrackerClass(which, 3, 5, 10, cpi, 10.0, fs=FS, fc=FC)
    ms, live = [], []
    for i, (d, f, s, ts) in enumerate(seq):
        tr.process(d, f, s, ts)
        tr.to_json(ts)
        if i >= warmup:
            ms.append((tr.ns_process + tr.ns_json) / 1e6)
            live.append(tr.get_n())
    tr.close()
    return dict(live_tracks=int(np.median(live)), ms=float(np.median(ms)), ms_max=float(max(ms)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpis", type=int, default=36)
    ap.add_argument("--warmup", type=int, default=24)
    ap.add_argument("--ref-max-adds", type=int, default=6000)
    a = ap.parse_args()
    import torch
    print(json.dumps(dict(device=torch.cuda.get_device_name(0))), flush=True)
    for cpi in (0.5, 0.75, 1.0):
        for ndet in (64, 256, 1024):
            nh = capi.tracker_plan(3, 5, 10, cpi, 10.0, FS, FC)[0]
            dro = run("dropin", ndet, cpi, a.cpis, a.warmup)
            r = dict(ndet=ndet, cpi=cpi, live_tracks=dro["live_tracks"], dropin_ms=dro["ms"],
                     dropin_ms_max=dro["ms_max"])
            if ndet * nh <= a.ref_max_adds and track_class.available("ref"):
                ref = run("ref", ndet, cpi, a.cpis, a.warmup)
                r.update(ref_ms=ref["ms"], speedup=ref["ms"] / dro["ms"])
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
