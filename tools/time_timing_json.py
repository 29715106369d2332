"""Time the timing stage (b200dd_pipeline_enable_timing_json) at config 2 (bench.py's geometry, spectrum and tracker
on): one pipeline with the stage on against one with it off, eager and graph-replayed, alternated over `rounds` rounds
in the same process.

Per CPI both pipelines make the same calls (submit_device, fetch, the track fetch); the one with the stage on also
fetches and commits its timing document, so the difference is the whole cost of the stage: the stamp kernels in the
chain, the stamps' read-back and the host render.  The time per CPI is a host clock around `steps` CPIs, each ending
in a synchronising fetch.  Also reported: the smallest nonzero difference between two stamps of one CPI seen over
the run (an upper bound of %globaltimer's update period, which is not measured here; the documents' 0.01 ms resolution
assumes it is well under 10 us), and the card's name and power limit.

    python tools/time_timing_json.py [--steps 40] [--rounds 7] [--out results/time_timing_json.json]
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

TRK = dict(M=3, N=5, delete=10, maxAcc=10, fc=204640000)


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


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
    min_step = [float("inf")]

    def cpi(p, timing, probe=False):
        ts[0] += 100
        p.fetch()
        p.fetch_track_json(ts[0])
        if timing:
            p.fetch_timing_json(ts[0])
        if timing and probe:  # outside the timed rounds
            _, v = p.timing_values()
            nz = v[v > 0]
            if nz.size:
                min_step[0] = min(min_step[0], float(nz.min()))

    rows = []
    for graph in (False, True):
        pipes = {}
        for on in (False, True):
            p = Pipeline(**bench.GEOM, clutter=bench.CLUTTER, detection=bench.DET, device=0, spectrum_bandwidth=2000,
                         tracker=TRK)
            if on:
                p.enable_timing_json(ts[0])
            if graph:  # the graph is recorded with the prepare's run, which is a CPI
                p.prepare_device(dx, dy)
            else:
                p.submit_device(dx, dy)
            cpi(p, on)
            pipes[on] = p

        def run(on, probe=False):
            p = pipes[on]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                p.submit_device(dx, dy)
                cpi(p, on, probe)
            return (time.perf_counter() - t0) / a.steps * 1e3

        ms = {False: [], True: []}
        run(False)
        run(True, probe=True)
        for _ in range(a.rounds):
            for on in (False, True):
                ms[on].append(run(on))
        med = {on: float(np.median(v)) for on, v in ms.items()}
        row = dict(geometry="config 2 (bench.py GEOM, CLUTTER, DET), spectrum + tracker", graph_replay=graph,
                   steps=a.steps, rounds=a.rounds, cpi_ms_stage_off=med[False], cpi_ms_stage_on=med[True],
                   added_ms=med[True] - med[False], ranges_off=[min(ms[False]), max(ms[False])],
                   ranges_on=[min(ms[True]), max(ms[True])], last_document=pipes[True].last_timing_doc.decode())
        print(json.dumps(row), flush=True)
        rows.append(row)
        for p in pipes.values():
            p.close()
    res = dict(gpu=gpu, rows=rows, smallest_nonzero_stage_ms=min_step[0], gpu_after=gpu_line())
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
