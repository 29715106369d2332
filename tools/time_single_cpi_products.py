"""BASELINE config 5 (ONE 4 s CPI @ 20 MS/s, N = 8e7, 512 x 4097 map, 410-tap clutter filter) with every product on
rank 0: SingleCpiPlan with a 2000-bin spectrum folded per rank slice and rank 0's importing pipeline
(Pipeline.submit_map) with detection and every document on.

    python tools/time_single_cpi_products.py [rounds] [--out DIR]                                      (1 GPU)
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/time_single_cpi_products.py

Prints one JSON line (rank 0):
- the GPU's name, power limit and max SM clock;
- ms per CPI of plan.run alone and of plan.run + submit_map + every fetch, alternated in rounds (median, range);
- device time of the slice fold (torch.profiler, written under --out) at the slice sizes of world 1, 2 and 8, as
  bytes/s at 8 B per sample, next to process_device's fold of the same number of samples (world 1 only);
- the device memory the config-5 importing pipeline takes (cudaMemGetInfo around its create)."""
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from blah2_b200.process import Ambiguity, Pipeline, SpectrumAnalyser, WienerHopfChunk
from blah2_b200.shard import Comm, SingleCpiPlan

GEOM = dict(delayMin=0, delayMax=511, dopplerMin=-512, dopplerMax=512, fs=20_000_000, nSamples=80_000_000)
CLUTTER = (-10, 400)
DET = dict(pfa=1e-5, nGuard=2, nTrain=6, minDelay=5, minDoppler=15.0, nCentroid=6)
BW = 2000.0


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def fold_kernel_ms(fn, reps, trace):
    """Mean device time per call of the fold kernels (spec_fold*) fn enqueues, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    if trace:
        prof.export_chrome_trace(trace)
    us = sum(e.device_time_total for e in prof.key_averages() if "spec_fold" in e.key)
    return us / reps / 1e3


def main():
    argv = sys.argv[1:]
    out = None
    if "--out" in argv:
        i = argv.index("--out")
        out = argv[i + 1]
        del argv[i:i + 2]
        os.makedirs(out, exist_ok=True)
    args = [a for a in argv if not a.startswith("--")]
    rounds = int(args[0]) if args else 5
    per_round = 3
    rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    comm = Comm(rank, world, local)
    n = GEOM["nSamples"]
    amb = Ambiguity(*GEOM.values(), True, device=local)
    whc = lambda a, b, nn, c0, nc: WienerHopfChunk(a, b, nn, c0, nc, device=local)  # noqa: E731
    bare = SingleCpiPlan(comm, amb, n, dev, clutter=CLUTTER, whc_factory=whc)
    pipe, pipe_bytes = None, 0
    if rank == 0:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(local)[0]
        pipe = Pipeline(**GEOM, roundHamming=True, clutter=CLUTTER, detection=DET, device=local, spectrum_bandwidth=BW,
                        map_json=True, maxhold=True, detection_json=True)
        pipe.enable_iqdata_json(0.0, -1.005, 1e21)
        pipe.enable_timing_json(int(time.time() * 1000))
        torch.cuda.synchronize()
        pipe_bytes = free0 - torch.cuda.mem_get_info(local)[0]
    spec = SpectrumAnalyser(n, BW, device=local)
    full = SingleCpiPlan(comm, amb, n, dev, clutter=CLUTTER, whc_factory=whc, spectrum=spec, pipeline=pipe)
    gen = torch.Generator(device="cuda").manual_seed(1234 + rank)
    x = torch.view_as_complex(torch.randn((bare.ns, 2), device="cuda", generator=gen)) * 1000.0
    y = 0.5 * x + 0.1 * torch.roll(x, 3) + torch.view_as_complex(torch.randn((bare.ns, 2), device="cuda", generator=gen)) * 10.0
    for p in (bare, full):
        p.x_own.copy_(x)
        p.y_own.copy_(y)
    del x, y
    s = torch.cuda.Stream()

    def run_bare():
        with torch.cuda.stream(s):
            bare.run(s)
        comm.sync()
        s.synchronize()

    def run_full():
        with torch.cuda.stream(s):
            full.run(s)
        comm.sync()
        s.synchronize()
        if pipe is not None:
            ts = int(time.time() * 1000)
            pipe.fetch()
            pipe.fetch_spectrum()
            pipe.fetch_map_json(ts)
            pipe.fetch_maxhold(ts)
            pipe.fetch_detection_json(ts)
            pipe.fetch_iqdata_json(ts)
            pipe.fetch_timing_json(ts)

    for _ in range(2):
        run_bare()
        run_full()
    times = {"run": [], "run_submit_fetch": []}
    for _ in range(rounds):
        for name, fn in (("run", run_bare), ("run_submit_fetch", run_full)):
            if world > 1:
                dist.barrier()
            t0 = time.perf_counter()
            for _ in range(per_round):
                fn()
            times[name].append((time.perf_counter() - t0) * 1e3 / per_round)
    timing_doc = None
    if pipe is not None:
        timing_doc = dict(zip(*pipe.timing_values()))
    line = {"config": "cfg5 single 4 s CPI @ 20 MS/s, 512 x 4097, WienerHopf 410 taps, 2000-bin spectrum, detection, "
                      "map / max-hold / detection / IQ-data / timing documents",
            "gpu": gpu_info(), "n_gpus": world, "rounds": rounds, "cpis_per_round": per_round}
    for name, v in times.items():
        line[f"ms_per_cpi_{name}"] = {"median": round(statistics.median(v), 3), "min": round(min(v), 3),
                                      "max": round(max(v), 3)}
    line["timing_document_ms"] = timing_doc
    line["importing_pipeline_device_bytes"] = int(pipe_bytes)
    if world == 1:
        folds = {}
        buf = torch.view_as_complex(torch.randn((n, 2), device="cuda")).contiguous()
        part = torch.empty(spec.nSpectrum, dtype=torch.complex128, device="cuda")
        for w in (1, 2, 8):
            m = n // w
            trace = os.path.join(out, f"fold_world{w}.pt.trace.json") if out else None
            ms = fold_kernel_ms(lambda: spec.fold_slice_device(buf[:m], 0, part), 20, trace)
            whole = SpectrumAnalyser(m, BW, device=local)
            ms_pd = fold_kernel_ms(lambda: whole.process_device(buf[:m]), 20, None)
            folds[f"world{w}"] = {"samples": m, "slice_fold_ms": round(ms, 4),
                                  "slice_fold_GBps": round(8 * m / ms / 1e6, 1),
                                  "process_device_fold_ms": round(ms_pd, 4),
                                  "process_device_fold_GBps": round(8 * m / ms_pd / 1e6, 1)}
            whole.close()
        line["fold"] = folds
    if rank == 0:
        print(json.dumps(line), flush=True)
        if out:
            with open(os.path.join(out, f"time_single_cpi_products_world{world}.json"), "w") as f:
                json.dump(line, f, indent=1)
    comm.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
