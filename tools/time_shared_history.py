"""Time a share set (b200dd_pipeline_share_history) against one unshared pipeline, at config 2 (bench.py's geometry)
with the spectrum, max-hold, detection JSON, IQ-data JSON and tracker stages on.

Per CPI both runs make the same calls: submit, fetch, then the documents of the four stateful stages (max-hold,
detection, IQ-data, track).  The unshared pipeline does submit -> fetch -> documents on one pipeline; the set of 3
submits CPI k on member k mod 3 and fetches CPI k - 2, so the set keeps 3 CPIs in flight and its max-hold push, history
commits and tracker update run at fetch time, ordered by the set's event.  A third run alternates 3 unshared
pipelines the same way: it overlaps CPIs as the set does, so set - alternated is the cost of sharing itself.  The time
per CPI is a host clock around `steps` CPIs ending in a synchronising fetch; the three runs are interleaved over
`rounds` rounds in the same process, eager and graph-replayed.

    python tools/time_shared_history.py [--steps 40] [--rounds 7] [--out results/time_shared_history.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from blah2_b200.process import Pipeline  # noqa: E402

MEMBERS = 3
TRK = dict(M=3, N=5, delete=10, maxAcc=10, fc=204640000)


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def _pipeline(bench):
    p = Pipeline(**bench.GEOM, clutter=bench.CLUTTER, detection=bench.DET, device=0, spectrum_bandwidth=2000,
                 maxhold=True, detection_json=True, tracker=TRK)
    p.enable_iqdata_json(0.0, 0.0, 0.0)
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    import bench
    from blah2_b200.scene import make_scene
    gpu = gpu_line()
    sc = make_scene(bench.N, bench.FS, seed=20260923)
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    ts = [1731000000000]

    def products(p):
        ts[0] += 100
        p.fetch()
        p.fetch_maxhold(ts[0])
        p.fetch_detection_json(ts[0])
        p.fetch_iqdata_json(ts[0])
        p.fetch_track_json(ts[0])

    rows = []
    for graph in (False, True):
        single = _pipeline(bench)
        members = [_pipeline(bench) for _ in range(MEMBERS)]
        Pipeline.share_history(members)
        alone = [_pipeline(bench) for _ in range(MEMBERS)]
        for p in [single] + members + alone:  # the graph is recorded with the prepare's run, which is a CPI
            if graph:
                p.prepare_device(dx, dy)
            else:
                p.submit_device(dx, dy)
            products(p)
        k = [0]

        def run_single():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                single.submit_device(dx, dy)
                products(single)
            return (time.perf_counter() - t0) / a.steps * 1e3

        def alternate(pipes):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(a.steps):  # in flight: the CPIs of all members; the oldest is fetched
                pipes[k[0] % MEMBERS].submit_device(dx, dy)
                k[0] += 1
                if i >= MEMBERS - 1:
                    products(pipes[(k[0] - MEMBERS) % MEMBERS])
            for j in range(MEMBERS - 1, 0, -1):
                products(pipes[(k[0] - j) % MEMBERS])
            return (time.perf_counter() - t0) / a.steps * 1e3

        runs = {"single": run_single, "shared": lambda: alternate(members), "alternated": lambda: alternate(alone)}
        ms = {name: [] for name in runs}
        for name, run in runs.items():
            run()
        for _ in range(a.rounds):
            for name, run in runs.items():
                ms[name].append(run())
        med = {name: float(np.median(v)) for name, v in ms.items()}
        row = dict(geometry="config 2 (bench.py GEOM), spectrum + max-hold + detection JSON + IQ-data JSON + tracker",
                   graph_replay=graph, members=MEMBERS, steps=a.steps, rounds=a.rounds,
                   cpi_ms_one_pipeline=med["single"], cpi_ms_shared=med["shared"],
                   cpi_ms_alternated_unshared=med["alternated"], added_ms_vs_one_pipeline=med["shared"] - med["single"],
                   added_ms_vs_alternated_unshared=med["shared"] - med["alternated"],
                   ranges={name: [min(v), max(v)] for name, v in ms.items()})
        print(json.dumps(row), flush=True)
        rows.append(row)
        for p in [single] + members + alone:
            p.close()
    res = dict(gpu=gpu, rows=rows, gpu_after=gpu_line())
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
