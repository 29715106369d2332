"""Diagnostic timing of the host-fed paths (never a source of bench numbers).

  python tools/time_e2e.py [steps]

For CPIs in flight = 1, 2, 4, 6, 8: ms per CPI of Pipeline.submit_host (complex128), submit_host_cf32 (complex64),
submit_host_rspduo (int16) and submit_host_ci8 (int8), beside the bare H2D copy of the same bytes from pinned memory
and the device-resident chain, so that what bounds the end-to-end number (PCIe, the kernels, or the host loop) can be
read off one table.  The GPU's name and power limit are printed with it.  The device chain is timed eager
and replayed as a CUDA graph (prepare_device); the host-fed legs run eager, as bench.py's e2e_rspduo_int16 does.
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from blah2_b200.process import Pipeline
from blah2_b200.scene import make_scene


def gpu_card():
    """The GPU's name and power limit as nvidia-smi reports them (None where it is not available)."""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return r.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def loop(pipes, submit, steps):
    n = len(pipes)
    for i in range(2 * n):
        submit(pipes[i % n], i)
        pipes[i % n].fetch()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        p = pipes[i % n]
        if i >= n:
            p.fetch()
        submit(p, i)
    for i in range(steps, steps + n):
        pipes[i % n].fetch()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def main(steps=24):
    N, FS = bench.N, bench.FS
    sc = make_scene(N, FS, seed=20260923)
    hx = [torch.from_numpy(np.roll(sc.x, 977 * b)).pin_memory() for b in range(2)]
    hy = [torch.from_numpy(np.roll(sc.y, 977 * b)).pin_memory() for b in range(2)]
    iq = np.empty((N, 4), dtype="<i2")
    iq[:, 0], iq[:, 1], iq[:, 2], iq[:, 3] = sc.x.real, sc.x.imag, sc.y.real, sc.y.imag
    hq = [torch.from_numpy(np.roll(iq, 977 * b, axis=0).copy()).pin_memory() for b in range(2)]
    # int8 and complex64 per channel (the scene's int16 values over 32, rounded to fit int8; the timing does not
    # depend on the values)
    i8 = [np.clip(np.round(np.stack([z.real, z.imag], axis=1) / 32.0), -128, 127).astype(np.int8) for z in (sc.x, sc.y)]
    h8 = [[torch.from_numpy(np.roll(c, 977 * b, axis=0).copy()).pin_memory() for c in i8] for b in range(2)]
    hf = [[torch.from_numpy(np.roll(z, 977 * b).astype(np.complex64)).pin_memory() for z in (sc.x, sc.y)]
          for b in range(2)]
    dx = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
    dy = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
    out = {}
    # bare H2D of one CPI's bytes from pinned memory
    dst = torch.empty(N * 4, dtype=torch.int16, device="cuda")
    dst2 = torch.empty(2 * N, dtype=torch.complex128, device="cuda")
    dst8 = torch.empty(2 * N, dtype=torch.int8, device="cuda")
    dstf = torch.empty(N, dtype=torch.complex64, device="cuda")
    out["gpu"] = gpu_card()
    for name, src, d in (("h2d_int16_16MB", hq[0].view(-1), dst),):
        for _ in range(3):
            d.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(20):
            d.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        out[name] = round((time.perf_counter() - t0) / 20 * 1e3, 4)
    for _ in range(3):
        dst2[:N].copy_(hx[0], non_blocking=True); dst2[N:].copy_(hy[0], non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(10):
        dst2[:N].copy_(hx[0], non_blocking=True); dst2[N:].copy_(hy[0], non_blocking=True)
    torch.cuda.synchronize()
    out["h2d_c128_64MB"] = round((time.perf_counter() - t0) / 10 * 1e3, 4)
    for name, (sx, sy), d in (("h2d_ci8_8MB", h8[0], dst8), ("h2d_cf32_32MB", hf[0], dstf)):  # both channels
        for _ in range(3):
            d.copy_(sx.view(-1), non_blocking=True); d.copy_(sy.view(-1), non_blocking=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(20):
            d.copy_(sx.view(-1), non_blocking=True); d.copy_(sy.view(-1), non_blocking=True)
        torch.cuda.synchronize()
        out[name] = round((time.perf_counter() - t0) / 20 * 1e3, 4)
    for npipe in (1, 2, 4, 6, 8):
        pipes = [Pipeline(**bench.GEOM, clutter=bench.CLUTTER, detection=bench.DET, device=0) for _ in range(npipe)]
        out[f"device_eager_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_device(dx, dy), steps), 4)
        for p in pipes:
            p.prepare_device(dx, dy)
        g = pipes[0].geometry
        hmaps = [torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex128).pin_memory() for _ in range(npipe)]
        idx = {id(p): k for k, p in enumerate(pipes)}
        out[f"device_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_device(dx, dy), steps), 4)
        out[f"int16_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_host_rspduo(hq[i % 2], map_out=hmaps[idx[id(p)]]), steps), 4)
        out[f"int16_nomap_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_host_rspduo(hq[i % 2]), steps), 4)
        out[f"ci8_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_host_ci8(*h8[i % 2], map_out=hmaps[idx[id(p)]]), steps), 4)
        out[f"ci8_nomap_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_host_ci8(*h8[i % 2]), steps), 4)
        out[f"cf32_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_host_cf32(*hf[i % 2], map_out=hmaps[idx[id(p)]]), steps), 4)
        out[f"cf32_nomap_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_host_cf32(*hf[i % 2]), steps), 4)
        out[f"c128_x{npipe}"] = round(loop(pipes, lambda p, i: p.submit_host(hx[i % 2], hy[i % 2], map_out=hmaps[idx[id(p)]]), steps), 4)
        for p in pipes:
            p.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:]))
