"""Time the max-hold document of blah2's /stash/map (blah2_b200/csrc/maxhold.cu) at the map sizes of BASELINE
configs 2, 3 and 5 with a full window of 20 CPIs:
  - push: CUDA events around many pushes (push + commit kernels) of a float2 map;
  - fetch: a host clock around the synchronous fetch (render kernels, device-to-host copy into pinned memory,
    header);
  - document bytes per cell, and the bytes each step must move (the byte model) over its time;
and, at config 2 (bench.py's geometry), the time per CPI of a graph-replayed pipeline with the stage on against one
with it off, alternated in the same process.  Maps: tests/maxhold_maps.py.

    python tools/time_maxhold.py [--iters 50] [--out results/time_maxhold.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from blah2_b200 import capi  # noqa: E402
from blah2_b200.process import MaxHold, Pipeline  # noqa: E402
from maxhold_maps import SEQS, seq_map  # noqa: E402

DEPTH = 20


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def kernel_ms(fetch, iters):
    """Summed device time per fetch of the render kernels (mh_len_kernel, scan_kernel, mh_write_kernel), from
    torch.profiler's CUDA activity over `iters` fetches."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fetch()
    us = sum(e.device_time_total for e in prof.key_averages()
             if any(k in e.key for k in ("mh_len_kernel", "scan_kernel", "mh_write_kernel")))
    return us / iters / 1e3


def handle_rows(iters):
    import torch
    lib = capi.load()
    rows = []
    for name in ("cfg2", "cfg3", "cfg5"):
        spec = SEQS[name]
        maps = []
        for i in range(DEPTH):
            m, delay, doppler = seq_map(spec, i)
            maps.append(torch.from_numpy(m).to("cuda", torch.complex64))
        metrics = (60.0, 320.0)
        mh = MaxHold(delay, doppler, spec["fs"], device=0)
        pinned = lib.b200dd_host_alloc(mh.max_bytes)
        st = torch.cuda.Stream()
        sp = C.c_void_p(st.cuda_stream)
        n = C.c_size_t()

        def push(i):
            capi.check(lib.b200dd_maxhold_push_device(mh._h, capi.ptr(maps[i % DEPTH]), 0, *metrics, sp))

        def fetch():
            capi.check(lib.b200dd_maxhold_fetch(mh._h, 1731000000000, C.c_void_p(pinned), mh.max_bytes, C.byref(n), sp))

        for i in range(2 * DEPTH):  # a full window, warm
            push(i)
        fetch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            for i in range(iters * 4):
                push(i)
            e1.record(st)
        e1.synchronize()
        push_ms = e0.elapsed_time(e1) / (iters * 4)
        tot = []
        for _ in range(iters):
            t0 = time.perf_counter()
            fetch()
            tot.append((time.perf_counter() - t0) * 1e3)
        fetch_ms = float(np.median(tot))
        kern = kernel_ms(fetch, iters)  # device time of the render kernels of one fetch
        cells = spec["nDop"] * spec["nDel"]
        doc = int(n.value)
        push_bytes = cells * (8 + 4)  # float2 cell read, int32 hundredths written
        render_bytes = cells * (DEPTH * 4 + 4 + 4) + doc  # window read, max written and read back, text written
        row = dict(map=name, cells=cells, doc_bytes=doc, doc_bytes_per_cell=doc / cells, push_ms=push_ms,
                   fetch_ms=fetch_ms, fetch_ms_min=float(np.min(tot)), render_kernels_ms=kern,
                   push_model_bytes=push_bytes, render_model_bytes=render_bytes,
                   push_gbps=push_bytes / push_ms / 1e6, render_kernels_gbps=render_bytes / kern / 1e6)
        print(json.dumps(row), flush=True)
        rows.append(row)
        lib.b200dd_host_free(C.c_void_p(pinned))
        mh.close()
        del maps
    return rows


def pipeline_row(steps, rounds):
    import torch
    import bench
    from blah2_b200.scene import make_scene
    sc = make_scene(bench.N, bench.FS, seed=20260923)
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    pipes = {}
    for on in (False, True):
        p = Pipeline(**bench.GEOM, clutter=bench.CLUTTER, detection=bench.DET, device=0, maxhold=on)
        p.prepare_device(dx, dy)
        p.fetch()
        pipes[on] = p

    def run(p):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            p.submit_device(dx, dy)
            p.fetch()
        return (time.perf_counter() - t0) / steps * 1e3

    for p in pipes.values():
        run(p)
    ms = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            ms[on].append(run(pipes[on]))
    off, on = float(np.median(ms[False])), float(np.median(ms[True]))
    row = dict(geometry="config 2 (bench.py GEOM)", graph_replay=True, steps=steps, rounds=rounds,
               cpi_ms_stage_off=off, cpi_ms_stage_on=on, added_ms=on - off,
               off_range=[min(ms[False]), max(ms[False])], on_range=[min(ms[True]), max(ms[True])])
    print(json.dumps(row), flush=True)
    for p in pipes.values():
        p.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    res = dict(gpu=gpu_line(), rows=handle_rows(a.iters), pipeline=pipeline_row(a.steps, a.rounds))
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
