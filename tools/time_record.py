"""Diagnostic timing of CPI records (never a source of bench numbers).

  python tools/time_record.py [reps]

For config 2 and a config-4-size geometry (N = 10^7, 512 x 1025; config 2's clutter window and detection):
  - the record's size in bytes, at 4096 detection slots, with and without the spectrum and timing stages;
  - the pack kernel's device time (torch.profiler, CUDA activities);
  - a graph-replayed submit_device followed by its fetch, export on and off, alternated in one loop (ms per CPI);
  - rank 0's cost per imported CPI at the config-4 size with every stage on: submit_record and every fetch, the host
    clock around each CPI, which ends synchronised;
  - from those, how many ranks one rank 0 keeps up with: a rank's graph-replayed CPI over rank 0's cost per CPI.
The GPU's name and power limit are printed with the numbers.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from blah2_b200.process import Pipeline
from tools.time_e2e import gpu_card

GEOMS = {
    "cfg2": dict(delayMin=0, delayMax=299, dopplerMin=-128, dopplerMax=128, fs=2_000_000, nSamples=2_000_000),
    "cfg4": dict(delayMin=0, delayMax=511, dopplerMin=-512, dopplerMax=512, fs=10_000_000, nSamples=10_000_000),
}
TRK = dict(M=2, N=3, delete=4, maxAcc=30, fc=204640000)
T_START = 1730999990000


def scene(g, seed):
    """A reference channel and two Doppler-shifted echoes of it, on the device."""
    N, fs = g["nSamples"], g["fs"]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    x = torch.randn(N, 2, device="cuda", generator=gen).view(torch.complex64).reshape(N) * 10
    y = torch.randn(N, 2, device="cuda", generator=gen).view(torch.complex64).reshape(N) * 3 + 8 * x
    t = torch.arange(N, device="cuda", dtype=torch.float64) / fs
    for d, f in ((37, 25.0), (120, -41.0)):
        y = y + 0.3 * torch.roll(x, d) * torch.exp(2j * np.pi * f * t).to(torch.complex64)
    x, y = x.contiguous(), y.contiguous()
    torch.cuda.synchronize()   # the pipelines read them on their own streams
    return x, y


def pipeline(geom, products=True, export=4096):
    kw = dict(roundHamming=True, device=0, clutter=bench.CLUTTER, detection=bench.DET, spectrum_bandwidth=2000)
    if products:
        kw.update(map_json=True, maxhold=True, detection_json=True, tracker=TRK, max_track_history=32)
    p = Pipeline(**GEOMS[geom], **kw)
    if products:
        p.enable_iqdata_json(-1.0, 1.0, 0.0)
    p.enable_timing_json(T_START)
    if export:
        p.enable_export(export)
    return p


def map_buf(p):
    g = p.geometry
    return torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")


def submit_times(geom, reps):
    """ms per graph-replayed submit_device + fetch, export off and on, alternated CPI by CPI."""
    x, y = scene(GEOMS[geom], 1)
    pipes = {False: pipeline(geom, products=False, export=None), True: pipeline(geom, products=False)}
    maps = {k: map_buf(p) for k, p in pipes.items()}
    for k, p in pipes.items():
        p.prepare_device(x, y, maps[k])
        p.fetch()
        for _ in range(3):
            p.submit_device(x, y, maps[k])
            p.fetch()
    acc = {False: 0.0, True: 0.0}
    for _ in range(reps):
        for k in (False, True):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipes[k].submit_device(x, y, maps[k])
            pipes[k].fetch()   # synchronises the pipeline's stream
            acc[k] += time.perf_counter() - t0
    return {("export_on" if k else "export_off"): round(v / reps * 1e3, 4) for k, v in acc.items()}


def pack_kernel_us(geom, reps):
    """pl_pack_kernel's mean device time over reps graph-replayed CPIs."""
    from torch.profiler import ProfilerActivity, profile
    x, y = scene(GEOMS[geom], 2)
    p = pipeline(geom, products=False)
    m = map_buf(p)
    p.prepare_device(x, y, m)
    p.fetch()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            p.submit_device(x, y, m)
            p.fetch()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "pl_pack_kernel" in e.name]
    return round(float(np.mean(times)), 3) if times else None, len(times)


def import_cost(geom, reps):
    """Rank 0's host time per imported CPI, every stage on: submit_record and every fetch (ms)."""
    e = pipeline(geom, products=False)
    q = pipeline(geom)
    recs, maps = [], []
    for i in range(4):
        x, y = scene(GEOMS[geom], 10 + i)
        m = map_buf(e)
        e.submit_device(x, y, m)
        torch.cuda.synchronize()
        recs.append(e.export_record().clone())
        maps.append(m)
        e.fetch()
    torch.cuda.synchronize()

    def one(i):
        ts = 1731000000000 + 100 * i
        q.submit_record(recs[i % 4], maps[i % 4])
        q.fetch()
        q.fetch_map_json(ts)
        q.fetch_spectrum()
        q.fetch_maxhold(ts)
        q.fetch_detection_json(ts)
        q.fetch_detection_stash()
        q.fetch_iqdata_json(ts)
        q.fetch_iqdata_stash()
        q.fetch_track_json(ts)
        q.fetch_timing_json(ts)
        q.fetch_timing_stash()
    for i in range(8):
        one(i)
    t0 = time.perf_counter()
    for i in range(8, 8 + reps):
        one(i)
    torch.cuda.synchronize()
    return round((time.perf_counter() - t0) / reps * 1e3, 4)


def main(reps=40):
    out = {"gpu": gpu_card(), "reps": reps}
    for geom in ("cfg2", "cfg4"):
        r = {}
        for ns, tm in ((True, True), (False, False)):
            kw = dict(roundHamming=True, device=0, clutter=bench.CLUTTER, detection=bench.DET)
            if ns:
                kw["spectrum_bandwidth"] = 2000
            p = Pipeline(**GEOMS[geom], **kw)
            if tm:
                p.enable_timing_json(T_START)
            r["record_bytes" + ("_spectrum_timing" if ns else "_bare")] = p.enable_export(4096)
            p.close()
        r["pack_kernel_us"], r["pack_kernels_seen"] = pack_kernel_us(geom, reps)
        r["graph_submit_fetch_ms"] = submit_times(geom, reps)
        out[geom] = r
    out["cfg4"]["import_all_fetches_ms"] = cost = import_cost("cfg4", reps)
    out["cfg4"]["ranks_per_rank0"] = round(out["cfg4"]["graph_submit_fetch_ms"]["export_on"] / cost, 2)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 40)
