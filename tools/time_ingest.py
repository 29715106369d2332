"""Device time of the int8 ingest kernel (pl_ingest_ci8_kernel) inside Pipeline.submit_host_ci8 (diagnostic, never a
source of bench numbers).

  python tools/time_ingest.py [reps]

For N = 2e6 and 2e7 instants: `reps` submits of pinned int8 buffers, recorded by torch.profiler with CUDA activities
(the kernel runs inside the submit, so no event can bracket it alone), and the kernel's mean device time with the
bytes it moves: 4 B read and 16 B written per instant.  Prints one JSON line with the GPU's name and power limit.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from blah2_b200.process import Pipeline
from time_e2e import gpu_card


def main(reps=20):
    out = {"gpu": gpu_card()}
    for n in (2_000_000, 20_000_000):
        # the ingest does not depend on the chain behind it: no filter, no detection, a small map
        pipe = Pipeline(0, 15, -8, 8, 2_000_000, n, roundHamming=False, device=0)
        rng = np.random.default_rng(7)
        bx, by = (torch.from_numpy(rng.integers(-128, 128, (n, 2), dtype=np.int8)).pin_memory() for _ in range(2))
        for _ in range(3):
            pipe.submit_host_ci8(bx, by)
            pipe.fetch()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                pipe.submit_host_ci8(bx, by)
                pipe.fetch()
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.events() if "pl_ingest_ci8_kernel" in e.name]
        pipe.close()
        assert len(us) == reps, f"{len(us)} kernel records for {reps} submits"
        t = float(np.mean(us))
        out[f"ci8_kernel_n{n}"] = {"us": round(t, 2), "min_us": round(float(np.min(us)), 2),
                                   "GB_per_s": round(20.0 * n / (t * 1e-6) / 1e9, 1)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:]))
