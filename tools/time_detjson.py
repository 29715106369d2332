"""Time the detection document and the /stash/detection history (blah2_b200/csrc/detjson.cu):
  - render: CUDA events around many renders (memset + dj_len_kernel + scan_kernel + dj_write_kernel) of a device
    list of 0, 64, 4096 and 2^18 detections;
  - stash fetch: a host clock around the synchronous fetch (table upload, render kernels, device-to-host copy into
    pinned memory) at 10^3, 10^5 and 10^6 held detections, and the render kernels' device time from torch.profiler;
and, at config 2 (bench.py's geometry), the time per CPI of a graph-replayed pipeline, submit -> fetch ->
fetch_detection_json, with the stage on against submit -> fetch with it off, alternated in the same process.

    python tools/time_detjson.py [--iters 50] [--out results/time_detjson.json]
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
from blah2_b200.process import DetectionJson, Pipeline  # noqa: E402
from detjson_lists import N_FULL, large_lists  # noqa: E402


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def render_rows(iters):
    import torch
    lib = capi.load()
    lists = [torch.from_numpy(a).cuda() for a in large_lists("bounded_full")]
    dj = DetectionJson(2000000, max_held=1 << 20, device=0)
    st = torch.cuda.Stream()
    sp = C.c_void_p(st.cuda_stream)
    rows = []
    for n in (0, 64, 4096, N_FULL):
        count = torch.tensor([n], dtype=torch.int32, device="cuda")

        def render():
            capi.check(lib.b200dd_detjson_render_device(dj._h, *(capi.ptr(a) for a in lists), capi.ptr(count), sp))

        for _ in range(3):
            render()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            for _ in range(iters):
                render()
            e1.record(st)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / iters
        doc = len(dj.fetch(1, stream=st.cuda_stream))
        row = dict(detections=n, render_ms=ms, doc_bytes=doc)
        print(json.dumps(row), flush=True)
        rows.append(row)
    dj.close()
    return rows


def stash_rows(iters):
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib = capi.load()
    per_doc = 1000
    v = [a[:per_doc] for a in large_lists("bounded_full")]
    dl, dp, sn = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in v)
    count = torch.tensor([per_doc], dtype=torch.int32, device="cuda")
    dj = DetectionJson(2000000, max_held=10 ** 6, device=0)
    pinned = lib.b200dd_host_alloc(dj.stash_max_bytes)
    n = C.c_size_t()

    def fetch():
        capi.check(lib.b200dd_detjson_fetch_stash(dj._h, C.c_void_p(pinned), dj.stash_max_bytes, C.byref(n), None))

    rows, docs = [], 0
    for held in (10 ** 3, 10 ** 5, 10 ** 6):
        while docs * per_doc < held:  # 1 ms apart: nothing is pruned
            dj.render_device(dl, dp, sn, count)
            dj.fetch(1731000000000 + docs)
            docs += 1
        fetch()
        tot = []
        for _ in range(iters):
            t0 = time.perf_counter()
            fetch()
            tot.append((time.perf_counter() - t0) * 1e3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                fetch()
        us = sum(e.device_time_total for e in prof.key_averages()
                 if any(k in e.key for k in ("ds_len_kernel", "scan_kernel", "ds_write_kernel")))
        row = dict(held=held, documents=docs, stash_bytes=int(n.value), fetch_ms=float(np.median(tot)),
                   fetch_ms_min=float(np.min(tot)), render_kernels_ms=us / iters / 1e3)
        print(json.dumps(row), flush=True)
        rows.append(row)
    lib.b200dd_host_free(C.c_void_p(pinned))
    dj.close()
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
        p = Pipeline(**bench.GEOM, clutter=bench.CLUTTER, detection=bench.DET, device=0, detection_json=on)
        p.prepare_device(dx, dy)
        p.fetch()
        if on:
            p.fetch_detection_json(0)
        pipes[on] = p
    ts = [1]

    def run(on):
        p = pipes[on]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            p.submit_device(dx, dy)
            p.fetch()
            if on:
                ts[0] += 100
                p.fetch_detection_json(ts[0])
        return (time.perf_counter() - t0) / steps * 1e3

    for on in pipes:
        run(on)
    ms = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            ms[on].append(run(on))
    off, on = float(np.median(ms[False])), float(np.median(ms[True]))
    row = dict(geometry="config 2 (bench.py GEOM)", graph_replay=True, steps=steps, rounds=rounds,
               detections_per_cpi=int(pipes[True].fetch()["detections"].get_nDetections()),
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
    res = dict(gpu=gpu_line(), render=render_rows(a.iters), stash=stash_rows(a.iters),
               pipeline=pipeline_row(a.steps, a.rounds))
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
