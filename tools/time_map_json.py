"""Time the map document of blah2.cpp:303-304 (Map::to_json + Map::delay_bin_to_km) at the map sizes of BASELINE
configs 2, 3 and 5: the device render (CUDA events around the body kernels, and around the kernels plus the
device-to-host copy of the bytes into pinned memory, header composition included) against the compiled
reference on one host core (oracle/_ref, where it was built).  Maps: tests/map_json_maps.py.

    python tools/time_map_json.py [--iters 50] [--out results/time_map_json.json]
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
from blah2_b200.process import MapJson  # noqa: E402
from map_json_maps import MAPS, hash_map  # noqa: E402


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def reference_ms(m, delay, doppler, noise, maxp, ts, fs, reps):
    from oracle import refjson
    if not refjson.available():
        return None
    lib = refjson.lib()
    m = np.ascontiguousarray(m)
    out = np.empty(m.size * 27 + (1 << 16), dtype=np.uint8)
    times = []
    for _ in range(reps):  # includes filling the reference Map from the array (one pass, small next to the text)
        t0 = time.perf_counter()
        lib.refjson_map_json(m.ctypes.data, m.shape[0], m.shape[1], delay.ctypes.data, doppler.ctypes.data, noise,
                             maxp, ts, fs, out.ctypes.data, out.size)
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--ref-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    lib = capi.load()
    rows = []
    for name in ("cfg2", "cfg3", "cfg5"):
        spec = MAPS[name]
        m, delay, doppler = hash_map(spec)
        noise, maxp = 66.0, 319.0
        mj = MapJson(delay, doppler, spec["fs"], device=0)
        d = torch.from_numpy(m).to("cuda", torch.complex64)
        pinned = lib.b200dd_host_alloc(mj.max_bytes)
        st = torch.cuda.Stream()
        sp = C.c_void_p(st.cuda_stream)
        n = C.c_size_t()

        def render():
            capi.check(lib.b200dd_mapjson_render_device(mj._h, capi.ptr(d), 0, noise, maxp, sp))

        def fetch():
            capi.check(lib.b200dd_mapjson_fetch(mj._h, spec["ts"], C.c_void_p(pinned), mj.max_bytes, C.byref(n), sp))

        for _ in range(5):
            render()
            fetch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            for _ in range(a.iters):
                render()
            e1.record(st)
        e1.synchronize()
        kern_ms = e0.elapsed_time(e1) / a.iters
        tot = []
        for _ in range(a.iters):
            t0 = time.perf_counter()
            render()
            fetch()
            tot.append((time.perf_counter() - t0) * 1e3)
        ref = reference_ms(m, delay, doppler, noise, maxp, spec["ts"], spec["fs"], a.ref_reps)
        row = dict(map=name, cells=int(m.size), bytes=int(n.value), bytes_per_cell=n.value / m.size,
                   render_kernels_ms=kern_ms, render_plus_d2h_ms=float(np.median(tot)), reference_ms=ref,
                   body_gbps=n.value / kern_ms / 1e6, hbm_bytes_per_cell_min=8 + n.value / m.size)
        print(json.dumps(row))
        rows.append(row)
        lib.b200dd_host_free(C.c_void_p(pinned))
        mj.close()
    res = dict(gpu=gpu_line(), rows=rows)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
