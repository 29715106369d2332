"""Time the device tracker per CPI -- Tracker::process on a device detection list plus the track document's fetch --
at config-like loads, and the reference's Tracker::process + Track::to_json on one host core
(oracle/_ref/libblah2tracker.so, where it was built) on the same sequence.

Each load is a sequence of CPIs of `ndet` detections at random positions outside the association window, with one
detection inside it every 12th CPI (every reached track then associates, and the ACTIVE ones coast into the
document).  M 3, N 5, delete 10, maxAcc 10, as config/config.yml; cpi 0.5 / 0.75 / 1 s gives 5 / 11 / 21 hypotheses
per detection, so the live tracks settle at tens to hundreds of thousands.  The first `--warmup` CPIs build the
state and are not timed.

    python tools/time_tracker.py [--cpis 36] [--warmup 24] [--no-ref] [--ref-max-adds 6000]

The reference's time grows with the live tracks (every CPI copies the whole Track, and the counts rescan every
track's state strings): it is timed only where ndet x hypotheses (the tracks each CPI adds) is at most --ref-max-adds.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from blah2_b200 import capi  # noqa: E402
from blah2_b200.process import Tracker  # noqa: E402
from oracle import reftracker  # noqa: E402

FS, FC = 2000000, 204640000


def sequence(ndet, n_cpi, cpi, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_cpi):
        d = rng.uniform(2, 400, ndet)
        f = rng.uniform(-300, 300, ndet)
        if i % 12 == 11:
            d[0], f[0] = 0.5, 0.25 / cpi
        out.append((d, f, rng.uniform(10, 30, ndet), 1731000000000 + int(1000 * cpi) * i))
    return out


def run(ndet, cpi, n_cpi, warmup, ref):
    import torch
    seq = sequence(ndet, n_cpi, cpi, seed=ndet)
    tr = Tracker(3, 5, 10, cpi, 10.0, FS, FC, max_tracks=1 << 20, max_history=24, device=0)
    dev = [[torch.from_numpy(a).cuda() for a in c[:3]] + [torch.tensor([ndet], dtype=torch.int32, device="cuda")]
           for c in seq]
    torch.cuda.synchronize()
    upd, tot, live, docb = [], [], [], []
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st = torch.cuda.current_stream().cuda_stream
    for i, (c, t) in enumerate(zip(seq, dev)):
        t0 = time.perf_counter()
        s0.record()
        tr.process_device(*t, c[3], stream=st)
        s1.record()
        doc = tr.fetch(c[3], stream=st)
        t1 = time.perf_counter()
        if i >= warmup:
            upd.append(s0.elapsed_time(s1))
            tot.append(1e3 * (t1 - t0))
            head = json.loads(doc[:doc.index(b',"data"')] + b"}")
            live.append(head["n"])
            docb.append(len(doc))
    tr.close()
    r = dict(ndet=ndet, cpi=cpi, live_tracks=int(np.median(live)), doc_bytes=int(np.median(docb)),
             doc_bytes_max=int(max(docb)), device_update_ms=float(np.median(upd)),
             device_update_and_fetch_ms=float(np.median(tot)), device_update_and_fetch_ms_max=float(max(tot)))
    if ref:
        rt = reftracker.RefTracker(3, 5, 10, cpi, 10.0, FS, FC)
        pr, js = [], []
        for i, c in enumerate(seq):
            rt.process(*c)
            if i >= warmup:
                pr.append(rt.ns_process / 1e6)
                js.append(rt.ns_json / 1e6)
        rt.close()
        r.update(ref_process_ms=float(np.median(pr)), ref_to_json_ms=float(np.median(js)))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpis", type=int, default=36)
    ap.add_argument("--warmup", type=int, default=24)
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--ref-max-adds", type=int, default=6000)
    a = ap.parse_args()
    import torch
    print(json.dumps(dict(device=torch.cuda.get_device_name(0))))
    ref = not a.no_ref and reftracker.available()
    for cpi in (0.5, 0.75, 1.0):
        for ndet in (64, 256, 1024):
            nh = capi.tracker_plan(3, 5, 10, cpi, 10.0, FS, FC)[0]
            print(json.dumps(run(ndet, cpi, a.cpis, a.warmup, ref and ndet * nh <= a.ref_max_adds)), flush=True)


if __name__ == "__main__":
    main()
