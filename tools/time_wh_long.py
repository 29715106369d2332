"""Per-stage device times of the clutter filter across tap counts, below and above 2048 taps.

    python tools/time_wh_long.py [--iters K] [--out DIR]

For each tap count (410, 2040, 2050, 3000, 4096) and CPI length (2e6, 2e7 samples): the correlation stage (K3), the
solve (K4) and the weight spectra + filter (K5), from CUDA events around each stage (b200dd_wh_profile_device) on
device-resident float2 IQ, median of K runs after 3 warm-ups, each run on a rolled copy of the scene.  Also prints
the plan (FFT length, lag blocks, partitions, solve threads) and the per-step solve latency (solve time / taps), and
the GPU's name, SM clock and power limit as the driver reports them.  Writes the table as JSON under --out.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from blah2_b200.process import WienerHopf
from blah2_b200.scene import make_scene

WINDOWS = {410: (-10, 400), 2040: (-10, 2030), 2050: (-50, 2000), 3000: (-50, 2950), 4096: (-96, 4000)}


def gpu_conditions():
    q = "name,clocks.sm,clocks.max.sm,power.limit,power.draw,temperature.gpu"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # the query is informational
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print("gpu:", torch.cuda.get_device_name(0), "|", gpu_conditions(), flush=True)
    rows = []
    for n in (2000000, 20000000):
        sc = make_scene(n, 2e6, seed=20261016)
        x0 = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
        y0 = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
        del sc
        xs = [torch.roll(x0, 977 * b) for b in range(4)]
        ys = [torch.roll(y0, 977 * b) for b in range(4)]
        yf = torch.empty_like(y0)
        for taps, (dm, dM) in WINDOWS.items():
            wh = WienerHopf(dm, dM, n)
            p = wh.plan
            s = torch.cuda.Stream()
            t = []
            with torch.cuda.stream(s):
                for i in range(args.iters + 3):
                    r = wh.profile_device(xs[i % 4], ys[i % 4], yf, s.cuda_stream)
                    if i >= 3:
                        t.append(r)
            s.synchronize()
            assert wh.last_status()
            c, so, a = (float(np.median([v[j] for v in t])) for j in range(3))
            row = dict(N=n, taps=taps, corr_ms=c, solve_ms=so, filter_ms=a, solve_step_ns=1e6 * so / taps,
                       corr_fft=p.corr_fft_len, corr_hop=p.corr_hop, lag_blocks=p.corr_lag_blocks,
                       filter_fft=p.filter_fft_len, filter_hop=p.filter_hop, partitions=p.filter_partitions,
                       solve_threads=p.solve_threads, solve_rows_per_thread=p.solve_rows_per_thread)
            rows.append(row)
            print(json.dumps(row), flush=True)
            del wh
        del xs, ys, x0, y0, yf
        torch.cuda.empty_cache()
    print("gpu after:", gpu_conditions(), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_wh_long.json"), "w") as f:
            json.dump(dict(gpu=torch.cuda.get_device_name(0), conditions=gpu_conditions(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
