"""Time the IQ-data document and the /stash/iqdata history (blah2_b200/csrc/iqjson.cu), at 2000 bins (blah2's
bandwidth at config 2) and at the 65536-bin bound:
  - render: CUDA events around many renders (memset + ij_len_kernel + scan_kernel + ij_write_kernel);
  - fetch: a host clock around the synchronous fetch of a rendered document into pinned memory (median);
  - stash fetch: a host clock around the synchronous fetch of a full 20-document history (median), and the render
    kernels' device time from torch.profiler;
and, at config 2 (bench.py's geometry) with the spectrum stage on, the time per CPI of a graph-replayed pipeline,
submit -> fetch -> fetch_iqdata_json with the stage on against submit -> fetch with it off, alternated in the same
process.

    python tools/time_iqjson.py [--iters 50] [--out results/time_iqjson.json]
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
from blah2_b200.process import IqDataJson, Pipeline  # noqa: E402
from iqjson_spectra import full_spectrum  # noqa: E402

METRICS = (0.0, 0.0, 0.0)


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def _median_ms(fn, iters):
    fn()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def handle_row(n, iters):
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib = capi.load()
    d = torch.from_numpy(full_spectrum()[:n].copy()).cuda()
    ij = IqDataJson(n, *METRICS, device=0)
    st = torch.cuda.Stream()
    sp = C.c_void_p(st.cuda_stream)

    def render():
        capi.check(lib.b200dd_iqjson_render_device(ij._h, capi.ptr(d), sp))

    for _ in range(3):
        render()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(st):
        e0.record(st)
        for _ in range(iters):
            render()
        e1.record(st)
    e1.synchronize()
    render_ms = e0.elapsed_time(e1) / iters
    pinned = lib.b200dd_host_alloc(ij.stash_max_bytes)
    nb = C.c_size_t()
    ts = [1731000000000]

    def fetch():  # render (not timed: it is enqueued before the clock starts) then the synchronous fetch
        ts[0] += 100
        capi.check(lib.b200dd_iqjson_fetch(ij._h, ts[0], C.c_void_p(pinned), ij.stash_max_bytes, C.byref(nb), sp))

    tot = []
    for i in range(iters + 1):
        render()
        st.synchronize()
        t0 = time.perf_counter()
        fetch()
        if i:
            tot.append((time.perf_counter() - t0) * 1e3)
    doc_bytes = int(nb.value)

    def fetch_stash():
        capi.check(lib.b200dd_iqjson_fetch_stash(ij._h, C.c_void_p(pinned), ij.stash_max_bytes, C.byref(nb), sp))

    stash_ms = _median_ms(fetch_stash, iters)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fetch_stash()
    us = sum(e.device_time_total for e in prof.key_averages()
             if any(k in e.key for k in ("is_len_kernel", "scan_kernel", "is_write_kernel")))
    row = dict(bins=n, render_ms=render_ms, doc_bytes=doc_bytes, fetch_ms=float(np.median(tot)),
               stash_documents=20, stash_bytes=int(nb.value), stash_fetch_ms=stash_ms,
               stash_render_kernels_ms=us / iters / 1e3)
    print(json.dumps(row), flush=True)
    lib.b200dd_host_free(C.c_void_p(pinned))
    ij.close()
    return row


def pipeline_row(steps, rounds):
    import torch
    import bench
    from blah2_b200.scene import make_scene
    sc = make_scene(bench.N, bench.FS, seed=20260923)
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    pipes = {}
    for on in (False, True):
        p = Pipeline(**bench.GEOM, clutter=bench.CLUTTER, detection=bench.DET, device=0, spectrum_bandwidth=2000)
        if on:
            p.enable_iqdata_json(*METRICS)
        p.prepare_device(dx, dy)
        p.fetch()
        if on:
            p.fetch_iqdata_json(0)
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
                p.fetch_iqdata_json(ts[0])
        return (time.perf_counter() - t0) / steps * 1e3

    for on in pipes:
        run(on)
    ms = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            ms[on].append(run(on))
    off, on = float(np.median(ms[False])), float(np.median(ms[True]))
    row = dict(geometry="config 2 (bench.py GEOM), spectrum stage on", graph_replay=True, steps=steps, rounds=rounds,
               bins=pipes[True].n_spectrum, cpi_ms_stage_off=off, cpi_ms_stage_on=on, added_ms=on - off,
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
    gpu = gpu_line()
    res = dict(gpu=gpu, handle=[handle_row(n, a.iters) for n in (2000, 65536)],
               pipeline=pipeline_row(a.steps, a.rounds), gpu_after=gpu_line())
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
