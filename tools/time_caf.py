"""Scratch timing of the device-resident CAF (CUDA events on torch's current stream)."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from blah2_b200.process import Ambiguity

CFGS = {
    "cfg1": (0, 299, -128, 128, 2000000, 2000000, True),
    "cfg3": (0, 511, -256, 256, 10000000, 20000000, True),
    "cfg4": (0, 511, -512, 512, 10000000, 10000000, True),
}

def _peak():
    """HBM bytes/s: MEASURED_PEAKS.json's hbm_gbs where it exists, else the H100 SXM data sheet's 3.35 TB/s."""
    try:
        return float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                 "MEASURED_PEAKS.json")))["hbm_gbs"]) * 1e9
    except (OSError, KeyError, ValueError):
        return 3350e9


PEAK = _peak()

def run(name, log2m=None, parts=None, iters=20, nbuf=8):
    if log2m: os.environ["B200DD_CAF_LOG2M"] = str(log2m)
    else: os.environ.pop("B200DD_CAF_LOG2M", None)
    if parts: os.environ["B200DD_CAF_PARTS"] = str(parts)
    else: os.environ.pop("B200DD_CAF_PARTS", None)
    geom = CFGS[name]
    amb = Ambiguity(*geom)
    g = amb.geometry
    n = geom[5]
    nbuf = max(2, min(nbuf, int(400e6 // (16 * n)) ))
    xs = [torch.randn(n, dtype=torch.complex64, device="cuda") for _ in range(nbuf)]
    ys = [torch.randn(n, dtype=torch.complex64, device="cuda") for _ in range(nbuf)]
    out = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    stream = torch.cuda.Stream()
    st = stream.cuda_stream
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        for i in range(3):
            amb.process_device(xs[i % nbuf], ys[i % nbuf], out, st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for i in range(iters):
            amb.process_device(xs[i % nbuf], ys[i % nbuf], out, st)
        e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    kr = []
    with torch.cuda.stream(stream):
        for i in range(10):
            kr.append(amb.profile_device(xs[i % nbuf], ys[i % nbuf], out, st))
    k_range = sum(a for a, _ in kr[2:]) / len(kr[2:])
    k_dop = sum(b for _, b in kr[2:]) / len(kr[2:])
    byts = 16 * g.n_used + 8 * g.n_doppler_bins * g.n_delay_bins
    print(json.dumps(dict(cfg=name, range_ms=round(k_range, 5), doppler_ms=round(k_dop, 5), log2m=g.range_fft_len, nseg=g.range_segments, parts=g.range_parts, hop=g.range_hop, m2=g.doppler_fft_len,
                          ms=round(ms, 4), maps_per_s=round(1e3 / ms, 1), msamples_per_s=round(n / ms / 1e3, 1),
                          gbs=round(byts / ms / 1e6, 1), frac=round(byts / (ms * 1e-3) / PEAK, 4))), flush=True)
    amb.close()

if __name__ == "__main__":
    sweep = "--sweep" in sys.argv
    for name in [a for a in sys.argv[1:] if not a.startswith("--")] or ["cfg1", "cfg3"]:
        run(name)
        if sweep:
            for l in (10, 11, 12, 13):
                for p in (1, 2, 4, 8):
                    run(name, l, p)
