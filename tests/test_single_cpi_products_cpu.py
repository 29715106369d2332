"""CPU: one CPI over GPUs with every product on one rank.

- The spectrum fold of a slice [sample0, sample0 + n) as spectrum.cu's kernels walk it (bands of nSpectrum samples,
  shifted by one for odd sample0 in the two-column kernel; whole bands unmasked, the first and last masked), restated
  in numpy: every read lies inside the slice's buffer, two-column loads stay 16-byte aligned, and the parts of any
  partition of [0, nfft) sum to the whole fold, whose finish is SpectrumAnalyser's spectrum.
- SingleCpiPlan with a spectrum and an importing pipeline at world 2 and 3 on gloo, with stand-ins that record calls.
- The new C entry points: declared, exported, argument checks without a device.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from blah2_b200 import capi
from blah2_b200.shard import SingleCpiPlan, TorchComm, block_range

FOLD_UNROLL = 8


# ---- the fold, restated -----------------------------------------------------------------------------------------
def phases(n_spec, dec):
    nfft = n_spec * dec
    k0 = nfft // 2 + 1
    t1 = np.exp(-2j * np.pi * ((k0 * np.arange(dec)) % dec) / dec)
    t2 = np.exp(-2j * np.pi * ((k0 * np.arange(n_spec)) % nfft) / nfft)
    return t1, t2


def fold_slice(x, sample0, n_spec, dec, vec2, want=4):
    """The part of x (x[0] = global sample sample0) as the kernels compute it: per chunk of bands, then summed."""
    t1, _ = phases(n_spec, dec)
    nfft = n_spec * dec
    n = len(x)
    end = min(sample0 + n, nfft)
    if end <= sample0:
        return np.zeros(n_spec, dtype=np.complex128)
    shift = sample0 & 1 if vec2 else 0
    qa, qb = (sample0 - shift) // n_spec, (end - shift + n_spec - 1) // n_spec
    fa, fb = (sample0 - shift + n_spec - 1) // n_spec, (end - shift) // n_spec
    rows = max(FOLD_UNROLL, -(-(qb - qa) // want))
    chunks = -(-(qb - qa) // rows)
    assert chunks <= want
    part = np.zeros(n_spec, dtype=np.complex128)
    k = np.arange(n_spec)
    for ch in range(chunks):
        q0 = qa + ch * rows
        q1 = min(qb, q0 + rows)
        lo = min(max(fa, q0), q1)
        hi = max(lo, min(fb, q1))
        acc = np.zeros(n_spec, dtype=np.complex128)
        for q in range(q0, q1):
            g = q * n_spec + shift + k              # the band's samples, column (shift + k) mod n_spec
            whole = lo <= q < hi
            ok = (g >= sample0) & (g < end)
            if whole:
                assert ok.all(), (q, sample0, end)
            if vec2:                                # a thread's pair starts at an even local offset
                assert ((g[0::2] - sample0) % 2 == 0).all()
            loc = g[ok] - sample0
            assert loc.min(initial=0) >= 0 and loc.max(initial=0) < n
            col = (shift + k[ok]) % n_spec
            row = g[ok] // n_spec
            assert (row < dec).all()
            np.add.at(acc, col, x[loc] * t1[row])
        part += acc
    return part


def finish(parts, n_spec, dec):
    _, t2 = phases(n_spec, dec)
    g = np.sum(np.asarray(parts).reshape(-1, n_spec), axis=0) * t2
    m = np.arange(n_spec)
    return np.exp(-2j * np.pi * np.outer(m, m) / n_spec) @ g


def spectrum_reference(x, n_spec, dec):
    """SpectrumAnalyser::process: the fft-shifted nfft-point spectrum of the first nfft samples, every dec-th bin."""
    nfft = n_spec * dec
    X = np.fft.fft(x[:nfft])
    k0 = nfft // 2 + 1
    return X[(np.arange(n_spec) * dec + k0) % nfft]


def cover(x, bounds, n_spec, dec, vec2):
    return [fold_slice(x[a:b], a, n_spec, dec, vec2) for a, b in zip(bounds[:-1], bounds[1:])]


GEOMS = [(8, 40), (9, 33), (2, 50), (64, 20)]


@pytest.mark.parametrize("n_spec,dec", GEOMS)
@pytest.mark.parametrize("vec2", [False, True])
def test_parts_of_any_partition_sum_to_the_whole_fold(n_spec, dec, vec2):
    if vec2 and n_spec % 2:
        pytest.skip("the two-column kernel needs an even nSpectrum")
    rng = np.random.default_rng(n_spec * 1000 + dec)
    nfft = n_spec * dec
    x = (rng.standard_normal(nfft + 7) + 1j * rng.standard_normal(nfft + 7)).astype(np.complex64).astype(np.complex128)
    whole = fold_slice(x, 0, n_spec, dec, vec2)
    ref = spectrum_reference(x, n_spec, dec)
    assert np.max(np.abs(finish([whole], n_spec, dec) - ref)) <= 1e-12 * np.max(np.abs(ref)) * nfft
    partitions = [
        [0, 3 * n_spec + 5, 7 * n_spec + 1, nfft + 7],                   # mid-row starts, odd and even
        [0, 4 * n_spec, 11 * n_spec, nfft],                              # row-aligned
        [0, 2 * n_spec + 1, 2 * n_spec + 3, nfft],                       # a slice inside one row
        [0, nfft - 3, nfft + 2, nfft + 7],                               # a slice past nfft
        [0, 5 * n_spec + 3, 5 * n_spec + 3, nfft],                       # an empty slice
        [0] + sorted(rng.choice(np.arange(1, nfft), 6, replace=False).tolist()) + [nfft],
    ]
    for b in partitions:
        parts = cover(x, b, n_spec, dec, vec2)
        assert np.max(np.abs(np.sum(parts, axis=0) - whole)) <= 1e-12 * max(np.max(np.abs(whole)), 1.0), b
    # a slice entirely past nfft, and an empty one, are zero parts
    assert not fold_slice(x[nfft:], nfft, n_spec, dec, vec2).any()
    assert not fold_slice(x[:0], 17, n_spec, dec, vec2).any()


def test_equal_batch_splits_of_a_cpi_with_samples_past_nfft():
    """SingleCpiPlan's slices: block_range of batches x nCorr, the last rank also the samples past them."""
    n_spec, dec, n_corr, n_dop = 20, 33, 13, 53
    n = n_dop * n_corr + 11
    nfft = n_spec * dec
    assert nfft <= n
    x = np.random.default_rng(3).standard_normal(n) + 0j
    whole = fold_slice(x, 0, n_spec, dec, True)
    for world in (2, 3, 8):
        parts = []
        for r in range(world):
            b0, nb = block_range(n_dop, r, world)
            s0 = b0 * n_corr
            ns = nb * n_corr + (n - n_dop * n_corr if r == world - 1 else 0)
            nf = max(0, min(ns, nfft - s0))
            parts.append(fold_slice(x[s0:s0 + nf], s0, n_spec, dec, r % 2 == 0))
        assert np.max(np.abs(np.sum(parts, axis=0) - whole)) <= 1e-12 * np.max(np.abs(whole))


# ---- SingleCpiPlan with stand-ins -------------------------------------------------------------------------------
class _Geom:
    def __init__(self, n_dop, n_del, n_corr):
        self.n_doppler_bins, self.n_delay_bins, self.n_corr = n_dop, n_del, n_corr


class _Amb:
    """Shapes of Ambiguity's stage-wise entry points; records the calls."""

    def __init__(self, geom, log):
        self.geometry, self.log = geom, log

    def range_device(self, x, y, b0, nb, R, stream=None):
        self.log.append(("range", b0, nb))
        R.copy_((x[:nb * self.geometry.n_corr].reshape(nb, -1)[:, :R.shape[1]]))

    def doppler_device(self, R, c0, nc, tile, stream=None):
        self.log.append(("doppler", c0, nc))
        tile.copy_(R[:, c0:c0 + nc])

    def place_tiles(self, tiles, n_tiles, m, stream=None):
        self.log.append(("place_tiles", n_tiles))


class _Spectrum:
    """SpectrumAnalyser's slice entry point on CPU tensors, by the restated fold."""

    def __init__(self, n_spec, dec, log):
        self.nSpectrum, self.decimation, self.nfft, self.log = n_spec, dec, n_spec * dec, log

    def fold_slice_device(self, d_x, sample0, d_part, stream=None):
        self.log.append(("fold", int(sample0), int(d_x.numel())))
        d_part.copy_(torch.from_numpy(fold_slice(d_x.numpy().astype(np.complex128), sample0, self.nSpectrum,
                                                 self.decimation, True)))


class _Pipeline:
    def __init__(self, log):
        self.log = log

    def stamp(self, slot, stream=None):
        self.log.append(("stamp", slot))

    def submit_map(self, d_map, d_status=None, d_parts=None, stream=None):
        self.log.append(("submit_map", d_status, None if d_parts is None else d_parts.numpy().copy()))


class _Chunk:
    """WienerHopfChunk's interface with a pass-through filter."""

    def __init__(self, delayMin, delayMax, nSamples, c0, nc):
        self.nBins, self.nc = 4, nc

    def halos(self):
        return 3, 2, 2

    def corr_device(self, x_loc, y_loc, ab, stream=None):
        ab.zero_()

    def filter_device(self, ab, x_loc, y_loc, y_out, stream=None):
        y_out.copy_(y_loc[:self.nc])

    def device_status(self):
        return 4242


N_SPEC, DEC, N_CORR, N_DOP, N_DEL = 12, 25, 10, 31, 6
N = N_DOP * N_CORR + 7


class _LogComm(TorchComm):
    def __init__(self, rank, world, log):
        super().__init__(rank, world)
        self.log = log

    def gather_async(self, send, recv, dst=0, after=None):
        self.log.append(("gather", int(send.numel())))
        super().gather_async(send, recv, dst, after)

    def gatherv_async(self, *a, **k):
        self.log.append(("gatherv",))
        super().gatherv_async(*a, **k)

    def allgatherv_async(self, *a, **k):
        self.log.append(("allgatherv",))
        super().allgatherv_async(*a, **k)


def _plan_worker(rank, world, port, products, clutter, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        log = []
        x = (np.random.default_rng(7).standard_normal(N) + 1j * np.random.default_rng(8).standard_normal(N))
        x = x.astype(np.complex64)
        spec = _Spectrum(N_SPEC, DEC, log) if products else None
        pipe = _Pipeline(log) if products and rank == 0 else None
        plan = SingleCpiPlan(_LogComm(rank, world, log), _Amb(_Geom(N_DOP, N_DEL, N_CORR), log), N, "cpu",
                             clutter=(0, 3) if clutter else None, whc_factory=_Chunk if clutter else None,
                             spectrum=spec, pipeline=pipe)
        plan.x_own.copy_(torch.from_numpy(x[plan.s0:plan.s0 + plan.ns]))
        for _ in range(2):
            plan.run(stream=None)
        q.put((rank, plan.s0, plan.ns, log))
    finally:
        dist.destroy_process_group()


def _run_plan(world, products, clutter, port):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_plan_worker, args=(r, world, port, products, clutter, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = dict((r, (s0, ns, log)) for r, s0, ns, log in (q.get(timeout=180) for _ in range(world)))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return out


def _strip(log):
    """The calls a plan without products makes."""
    return [e for e in log if e[0] not in ("fold", "stamp", "submit_map") and e != ("gather", N_SPEC)]


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("clutter", [False, True])
def test_single_cpi_plan_products_gloo(world, clutter):
    port = 31000 + (os.getpid() % 1500) + 10 * world + clutter
    base = _run_plan(world, False, clutter, port)
    got = _run_plan(world, True, clutter, port + 3)
    x = (np.random.default_rng(7).standard_normal(N) + 1j * np.random.default_rng(8).standard_normal(N))
    x = x.astype(np.complex64).astype(np.complex128)
    nfft = N_SPEC * DEC
    oracle = finish([fold_slice(x, 0, N_SPEC, DEC, True)], N_SPEC, DEC)
    for r in range(world):
        s0, ns, log = got[r]
        # without the new arguments the calls are the plan's own; with them, only the new ones are added
        assert _strip(log) == base[r][2]
        assert not any(e[0] in ("fold", "stamp", "submit_map") for e in base[r][2])
        folds = [e for e in log if e[0] == "fold"]
        a, b = s0, min(s0 + ns, nfft)
        assert folds == [("fold", s0, max(0, b - a))] * 2
        if r != 0:
            assert not any(e[0] in ("stamp", "submit_map") for e in log)
            continue
        for k in range(2):  # each run: CHAIN < SPECTRUM < CLUTTER < submit_map, once
            run = log[[i for i, e in enumerate(log) if e == ("stamp", capi.STAMP_CHAIN)][k]:]
            names = [e[0] if e[0] != "stamp" else ("stamp", e[1]) for e in run]
            i_chain, i_spec, i_clut = (names.index(("stamp", s)) for s in
                                       (capi.STAMP_CHAIN, capi.STAMP_SPECTRUM, capi.STAMP_CLUTTER))
            i_sub = names.index("submit_map")
            assert i_chain < names.index("fold") < i_spec < i_clut < names.index("range") < i_sub
            assert names.count("submit_map") == (1 if k == 1 else 2)
        subs = [e for e in log if e[0] == "submit_map"]
        assert len(subs) == 2
        for _, status, parts in subs:
            assert status == (4242 if clutter else None)
            assert parts.shape == (world, N_SPEC)
            for rr in range(world):  # rank order
                s0r, nsr, _ = got[rr]
                nf = max(0, min(nsr, nfft - s0r))
                np.testing.assert_allclose(parts[rr], fold_slice(x[s0r:s0r + nf], s0r, N_SPEC, DEC, True),
                                           rtol=0, atol=1e-12)
            spec = finish(parts, N_SPEC, DEC)
            assert np.max(np.abs(spec - oracle)) <= 1e-12 * np.max(np.abs(oracle))


# ---- C ABI ------------------------------------------------------------------------------------------------------
def test_new_entry_points_declared_and_exported():
    lib = C.CDLL(capi.LIB_PATH)
    names = {n for n, _, _ in capi.SIGNATURES}
    for name in ("b200dd_spectrum_fold_slice_device", "b200dd_spectrum_finish_device", "b200dd_pipeline_submit_map",
                 "b200dd_pipeline_stamp"):
        assert name in names and hasattr(lib, name)
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200dd.h")).read()
    for k, v in (("CHAIN", capi.STAMP_CHAIN), ("SPECTRUM", capi.STAMP_SPECTRUM), ("CLUTTER", capi.STAMP_CLUTTER)):
        assert f"#define B200DD_STAMP_{k} {v} " in text


def test_null_handles_and_no_device():
    lib = capi.load()
    buf = (C.c_double * 8)()
    assert lib.b200dd_spectrum_fold_slice_device(None, buf, 0, 4, buf, None) == capi.ERR_ARG
    assert lib.b200dd_spectrum_finish_device(None, buf, 1, None, None) == capi.ERR_ARG
    assert lib.b200dd_pipeline_submit_map(None, buf, None, None, 0, None) == capi.ERR_ARG
    assert lib.b200dd_pipeline_stamp(None, capi.STAMP_CHAIN, None) == capi.ERR_ARG
    if capi.device_count() > 0:
        return
    h = C.c_void_p()
    assert lib.b200dd_spectrum_create(80000000, 2000.0, -1, C.byref(h)) == capi.ERR_CUDA
    p = capi.PipelineParams()
    p.caf = capi.CafParams(-10, 300, -300, 300, 2000000, 1000000, 1, -1)
    assert lib.b200dd_pipeline_create(C.byref(p), C.byref(h)) == capi.ERR_CUDA
