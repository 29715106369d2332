"""GPU: one CPI over GPUs with every product on one rank.

- The spectrum of slices: one slice [0, n) and a one-part finish equal b200dd_spectrum_process_device bit for bit;
  the parts of slices covering [0, nfft) (equal batch splits, mid-row, odd and single-row boundaries, 8- and 16-byte
  aligned buffers) give the spectrum, the same on every run.
- b200dd_pipeline_submit_map: a pipeline given another pipeline's map, clutter-filter verdict and the spectrum part
  of the CPI gives every product that pipeline gives, over a scene sequence with a failed solve, alone and as two
  share-set members; SingleCpiPlan at world size 1 with a spectrum and an importing pipeline; every refused call
  enqueues nothing.
"""
import json
import math
import os

import numpy as np
import pytest

from blah2_b200 import capi
from blah2_b200.process import Ambiguity, IqDataJson, Pipeline, SpectrumAnalyser, WienerHopfChunk
from blah2_b200.shard import Comm, SingleCpiPlan, block_range
from blah2_b200.scene import random_iq
from oracle import blah2_oracle as O
from spectrum_cases import ROWS, row_id
from test_spectrum_envelope_gpu import U, error_bar, make_input
from test_record_gpu import BAD, GEOMS, METRICS, N_CPI, _map_buf, _pipeline, _products, _scenes, _ts

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

torch = pytest.importorskip("torch")


def _bits(t):
    return torch.view_as_real(t).contiguous().view(torch.int64)


def _x(n, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    x = torch.randn(n + 1, 2, device="cuda", generator=g).view(torch.complex64).reshape(n + 1) * 7
    torch.cuda.synchronize()  # the handles run on their own streams
    return x


@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_one_slice_equals_process_device(row):
    sa = SpectrumAnalyser(row["n"], row["bw"], device=0)
    n, ns = row["n"], sa.nSpectrum
    buf = _x(n, 5 + ns)
    for x in (buf[:n], buf[1:]):  # 16- and 8-byte aligned
        ref = torch.empty(ns, dtype=torch.complex128, device="cuda")
        got = torch.empty_like(ref)
        part = torch.empty((1, ns), dtype=torch.complex128, device="cuda")
        sa.process_device(x, ref)
        sa.fold_slice_device(x, 0, part[0])
        sa.finish_device(part, got)
        torch.cuda.synchronize()
        assert torch.equal(_bits(got), _bits(ref)), (row, x.data_ptr() % 16)


def _partitions(n, nfft, n_spec, n_dop, n_corr):
    out = {}
    for k in (2, 3, 8):  # SingleCpiPlan's slices: batches x nCorr, the last one up to n
        b = [block_range(n_dop, r, k)[0] * n_corr for r in range(k)] + [n]
        out[f"batches{k}"] = b
    q = nfft // n_spec
    out["adversarial"] = [0, 3 * n_spec + 5, 3 * n_spec + 7, 7 * n_spec, (q // 2) * n_spec + 1, nfft - 3, n]
    out["odd"] = [0, 1, 2 * n_spec + 3, 5 * n_spec + 2 * n_spec // 3 * 2 + 1, n]
    # an odd start whose masked first band, wrap column and masked last band all lie in one chunk of the fold
    out["odd_one_chunk"] = [0, 4 * n_spec + 3, 7 * n_spec + 12, n]
    return out


def _slice_input(buf, a, b, aligned16):
    """buf[a:b] at a 16-byte-aligned address (a fresh copy) or at one 8 bytes past it; the alignment picks the fold
    kernel (two columns per thread on 16 bytes and an even bin count, one column on 8 bytes)."""
    if aligned16:
        x = buf[a:b].clone()
        assert b == a or x.data_ptr() % 16 == 0
    else:
        tmp = torch.empty(b - a + 1, dtype=torch.complex64, device="cuda")
        tmp[1:] = buf[a:b]
        x = tmp[1:]
        assert b == a or x.data_ptr() % 16 == 8
    torch.cuda.synchronize()  # the copy (torch's stream) is done before the handle's stream reads it
    return x


def _fold_partition(sa, buf, b, aligned16):
    k = len(b) - 1
    parts = torch.empty((k, sa.nSpectrum), dtype=torch.complex128, device="cuda")
    xs = [_slice_input(buf, b[r], b[r + 1], aligned16(r)) for r in range(k)]
    for r in range(k):
        sa.fold_slice_device(xs[r], b[r], parts[r])
    out = torch.empty(sa.nSpectrum, dtype=torch.complex128, device="cuda")
    sa.finish_device(parts, out)
    torch.cuda.synchronize()
    return parts, out


def _slice_bar(r, geom, x, k):
    """The FP64 envelope of tests/test_spectrum_envelope_gpu.py widened by the additions slices add: a slice's chunk
    reduction (32 warps and its chunks) and the k - 1 additions of the parts."""
    extra = (k - 1) + 32 + math.ceil(int(geom.fold_chunks) / 32)
    return error_bar(r, geom, x) + 2 * U * math.sqrt(extra) * float(np.sum(np.abs(x[:r["nfft"]].astype(np.complex128))))


@pytest.mark.parametrize("geom", ["cfg2", "cfg4"])
def test_slices_sum_to_the_spectrum(geom):
    """Slices of the envelope test's input (noise under a strong tone and DC) at config 2 and the config-4 size.  Odd
    starts fold from 16-byte-aligned copies, so they run the two-column kernel that pairs columns (2j+1, 2j+2); the
    other slices alternate between the two kernels.  Every bin lies within the widened FP64 envelope of numpy's
    spectrum, a repeated run is bit-identical, and an odd slice's part is the same whichever kernel folds it."""
    g = GEOMS[geom]
    n = g["nSamples"]
    caf, _, _ = capi.caf_plan(g["delayMin"], g["delayMax"], g["dopplerMin"], g["dopplerMax"], g["fs"], n, True)
    sa = SpectrumAnalyser(n, 2000.0, device=0)
    ns, dec, nfft = sa.nSpectrum, sa.decimation, sa.nfft
    row = dict(n=n, bw=2000.0, n_spectrum=ns, dec=dec, nfft=nfft)
    x_np, _ = make_input(row, seed=ns + dec)
    assert nfft == n  # no NaN past nfft reaches a slice
    ref, _ = O.spectrum_process(x_np.astype(np.complex128), n, 2000.0)
    buf = torch.from_numpy(x_np).cuda()
    torch.cuda.synchronize()
    for name, b in _partitions(n, nfft, ns, caf.n_doppler_bins, caf.n_corr).items():
        k = len(b) - 1
        if name.startswith(("odd", "adversarial")):
            assert any(b[r] % 2 for r in range(1, k)), name
        pick = lambda r: b[r] % 2 == 1 or r % 2 == 0  # noqa: E731
        runs = [_fold_partition(sa, buf, b, pick) for _ in range(2)]
        assert torch.equal(_bits(runs[0][1]), _bits(runs[1][1])), name
        got = runs[0][1].cpu().numpy()
        err = np.abs(got - ref)
        bar = _slice_bar(row, sa.geometry, x_np, k)
        assert float(err.max()) <= bar, (name, float(err.max() / bar))
        # the same odd slices folded by the one-column kernel: the same sums, grouped differently
        other, _ = _fold_partition(sa, buf, b, lambda r: False)
        for r in range(k):
            if b[r] % 2:
                d = float((other[r] - runs[0][0][r]).abs().max())
                assert d <= 1e-13 * float(runs[0][0][r].abs().max()), (name, r, d)


@pytest.mark.parametrize("name", ["spectrum_a", "spectrum_b", "spectrum_c", "spectrum_d"])
def test_slices_against_the_reference_golden(name):
    """The golden spectra of the compiled reference (tests/golden/spectrum_*.npz) from three slices with odd and
    mid-row boundaries.  The slices take float32 samples and the golden input is complex128, so the spectrum of the
    rounding (numpy FP64, linear in x) is added to the golden one; what is left is the 1e-11 bar of
    tests/test_spectrum_gpu.py."""
    d = np.load(os.path.join(GOLD, name + ".npz"))
    n, bw, seed = int(d["params"][0]), float(d["params"][1]), int(d["params"][2])
    x64, _ = random_iq(n, seed)
    x32 = x64.astype(np.complex64)
    sa = SpectrumAnalyser(n, bw, device=0)
    ns, nfft = sa.nSpectrum, sa.nfft
    delta, _ = O.spectrum_process(x32.astype(np.complex128) - x64, n, bw)
    want = d["spectrum"] + delta
    buf = torch.from_numpy(x32).cuda()
    torch.cuda.synchronize()
    a = min(ns + 3, nfft - 2) | 1
    bounds = [0, a, max(a, nfft - ns // 2 - 1), n]
    for aligned in (True, False):
        _, out = _fold_partition(sa, buf, bounds, lambda r: aligned)
        got = out.cpu().numpy()
        scale = float(np.max(np.abs(d["spectrum"])))
        assert float(np.max(np.abs(got - want))) <= 1e-11 * scale, (name, aligned)


def _verdict(fail):
    return torch.tensor([capi.FILTER_FAILED if fail else 0], dtype=torch.int32, device="cuda")


def _doc_keys(tm):
    return list(tm) if isinstance(tm, dict) else tm


@pytest.mark.parametrize("members", [1, 2])
def test_submit_map_equals_the_pipeline_that_ran_the_cpi(members):
    """Pipeline A runs every CPI (submit_device); pipeline B (or two share-set members) takes A's map, A's verdict and
    the spectrum part of one slice of the CPI.  23+ CPIs: the max-hold window wraps; CPI BAD fails its solve."""
    geom = "cfg2"
    a = _pipeline(geom)
    bs = [_pipeline(geom) for _ in range(members)]
    if members > 1:
        Pipeline.share_history(bs)
    sa = SpectrumAnalyser(GEOMS[geom]["nSamples"], 2000.0, device=0)
    m = _map_buf(a)
    keep = []
    for i, (x, y) in enumerate(_scenes(geom)):
        a.submit_device(x, y, m)
        torch.cuda.synchronize()
        pa, tma = _products(a, i)
        failed = pa[0][1][1] != capi.OK
        assert failed == (i == BAD)
        part = torch.empty((1, sa.nSpectrum), dtype=torch.complex128, device="cuda")
        sa.fold_slice_device(x, 0, part[0])
        mb = m.clone()
        st = _verdict(failed)
        keep.append((mb, st, part))
        torch.cuda.synchronize()  # the part (the handle's stream), the map copy and the verdict (torch's) are written
        b = bs[i % members]
        b.submit_map(mb, st.data_ptr(), part)
        pb, tmb = _products(b, i)
        assert pb == pa, i
        assert _doc_keys(tmb) == _doc_keys(tma), i
    assert N_CPI >= 23
    for p in [a] + bs:
        p.close()


def _stagewise_map(amb, x, y, k, out):
    """K ranks emulated on one device: range rows, Doppler tiles, tile placement."""
    g = amb.geometry
    R = torch.empty((g.n_doppler_bins, g.n_delay_bins), dtype=torch.complex64, device="cuda")
    for r in range(k):
        b0, nb = block_range(g.n_doppler_bins, r, k)
        lo, hi = b0 * g.n_corr, (b0 + nb) * g.n_corr
        amb.range_device(x[lo:hi], y[lo:hi], b0, nb, R[b0:b0 + nb])
    tiles = []
    for r in range(k):
        c0, nc = block_range(g.n_delay_bins, r, k)
        t = torch.empty((g.n_doppler_bins, nc), dtype=torch.complex64, device="cuda")
        amb.doppler_device(R, c0, nc, t)
        tiles.append(t.reshape(-1))
    torch.cuda.synchronize()  # the handle's stream wrote the tiles
    amb.place_tiles(torch.cat(tiles), k, out)


@pytest.mark.parametrize("k", [2, 3])
def test_emulated_ranks_without_filter(k):
    geom = "cfg2"
    g = GEOMS[geom]
    a = _pipeline(geom, clutter=None)
    b = _pipeline(geom, clutter=None)
    amb = Ambiguity(g["delayMin"], g["delayMax"], g["dopplerMin"], g["dopplerMax"], g["fs"], g["nSamples"], True,
                    device=0)
    sa = SpectrumAnalyser(g["nSamples"], 2000.0, device=0)
    ij = IqDataJson(sa.nSpectrum, *METRICS, device=0)
    n, gm = g["nSamples"], amb.geometry
    ma, mb = _map_buf(a), _map_buf(b)
    differing = 0
    for i, (x, y) in enumerate(_scenes(geom)[:6]):
        a.submit_device(x, y, ma)
        torch.cuda.synchronize()
        pa, _ = _products(a, i)
        _stagewise_map(amb, x, y, k, mb)
        bounds = [block_range(gm.n_doppler_bins, r, k)[0] * gm.n_corr for r in range(k)] + [n]
        parts = torch.empty((k, sa.nSpectrum), dtype=torch.complex128, device="cuda")
        for r in range(k):
            hi = min(bounds[r + 1], sa.nfft)
            sa.fold_slice_device(x[bounds[r]:max(hi, bounds[r])], bounds[r], parts[r])
        torch.cuda.synchronize()
        assert torch.equal(mb, ma), i
        b.submit_map(mb, None, parts)
        pb, _ = _products(b, i)
        da, db = dict(pa), dict(pb)
        for name in ("fetch", "map", "maxhold", "detection", "detection_stash", "track"):
            assert da[name] == db[name], (i, name)
        spec = torch.from_numpy(np.frombuffer(db["spectrum"], dtype=np.complex128).copy()).cuda()
        ij.render_device(spec)
        assert ij.fetch(_ts(i)) == db["iqdata"], i
        va = json.loads(da["iqdata"])["spectrum"]
        vb = json.loads(db["iqdata"])["spectrum"]
        diff = [j for j in range(len(va)) if va[j] != vb[j]]
        differing += len(diff)
        sref = np.frombuffer(da["spectrum"], dtype=np.complex128)
        for j in diff:  # a bin whose text differs sits on a 0.01 boundary of 10 log10 |s|, within the FP64 envelope
            v = 10 * np.log10(abs(sref[j]))
            assert abs(v * 100 - np.round(v * 100)) < 1e-6, (i, j, va[j], vb[j])
    print(f"k={k}: {differing} IQ-data bins differ in text over 6 CPIs")


def _chunked_filter(x, y, clutter, k, rank_one=False):
    """The clutter filter of one CPI emulated over k chunks on one device, as tests/test_wh_gpu.py's
    test_chunked_filter_emulating_several_ranks does: per-chunk correlations, their sum (the all-reduce), the
    replicated solve and per-chunk filter.  rank_one: the summed reference correlations are replaced by a[k] = 2 for
    every k, whose Toeplitz matrix 2 u u^H is rank one (the solve must fail).  Returns the chunk handles and the
    filtered surveillance channel."""
    n = x.numel()
    chunks, abs_ = [], []
    for r in range(k):
        c0, nc = block_range(n, r, k)
        ch = WienerHopfChunk(clutter[0], clutter[1], n, c0, nc, device=0)
        xl, xr, yr = ch.halos()
        ix = torch.arange(c0 - xl, c0 + nc + xr, device="cuda") % n
        iy = torch.arange(c0, c0 + nc + yr, device="cuda") % n
        x_loc, y_loc = x[ix].contiguous(), y[iy].contiguous()
        ab = torch.zeros(2 * ch.nBins, dtype=torch.complex128, device="cuda")
        torch.cuda.synchronize()
        ch.corr_device(x_loc, y_loc, ab)
        torch.cuda.synchronize()
        chunks.append((ch, x_loc, y_loc, nc))
        abs_.append(ab)
    ab_sum = torch.stack(abs_).sum(0)
    if rank_one:
        ab_sum[:chunks[0][0].nBins] = 2.0
    outs = []
    torch.cuda.synchronize()
    for ch, x_loc, y_loc, nc in chunks:
        o = torch.empty(nc, dtype=torch.complex64, device="cuda")
        ch.filter_device(ab_sum, x_loc, y_loc, o)
        outs.append(o)
    torch.cuda.synchronize()
    return [c[0] for c in chunks], torch.cat(outs)


def test_chunked_filter_verdict_into_submit_map(relerr):
    """The clutter filter over K = 3 emulated chunks and the CAF over 3 emulated ranks; the import takes the verdict
    from a chunk handle's status word.  The map meets the 1e-5 bar of the oracle, the detection list equals
    b200dd_det_process_device on the same map and the map document b200dd_mapjson_render_device's.  A rank-one
    reference correlation (the system of tests/test_wh_conditioning_gpu.py's singular cases, which the solve must
    reject) imports as a failed solve: nothing is committed and nCpi does not step."""
    from blah2_b200.process import MapJson, _DetHandle
    from blah2_b200.scene import make_scene
    geom = (-5, 60, -200, 200, 100000, 100000)
    clutter = (-4, 40)
    det = dict(pfa=1e-4, nGuard=2, nTrain=6, minDelay=3, minDoppler=15.0, nCentroid=4)
    fs, n = geom[4], geom[5]
    p = Pipeline(*geom, roundHamming=True, clutter=clutter, detection=det, device=0, map_json=True,
                 detection_json=True)
    p.enable_timing_json(1730999990000)
    amb = Ambiguity(*geom, True, device=0)
    gm = amb.geometry
    dh = _DetHandle(det["pfa"], det["nGuard"], det["nTrain"], det["minDelay"], det["minDoppler"], det["nCentroid"],
                    det["nCentroid"], 1.0 / (n / fs), True, True, gm.n_doppler_bins, gm.n_delay_bins, device=0)
    mj = MapJson(p.delay, p.doppler, fs, device=0)
    m = torch.empty((gm.n_doppler_bins, gm.n_delay_bins), dtype=torch.complex64, device="cuda")
    n_cpi = []
    for i in range(3):
        sc = make_scene(n, fs, seed=21 + i, n_clutter=8)
        x = torch.from_numpy(sc.x.astype(np.complex64)).cuda()
        y = torch.from_numpy(sc.y.astype(np.complex64)).cuda()
        torch.cuda.synchronize()
        failed = i == 1
        chunks, yf = _chunked_filter(x, y, clutter, 3, rank_one=failed)
        assert [c.last_status() for c in chunks] == [not failed] * 3
        _stagewise_map(amb, x, yf, 3, m)
        torch.cuda.synchronize()
        p.submit_map(m, chunks[0].device_status())
        ts = 1731000000000 + 100 * i
        res = p.fetch()
        if failed:
            assert res["skipped"]
            stash = p.fetch_detection_stash()
            for f in (lambda: p.fetch_map_json(ts), lambda: p.fetch_detection_json(ts), lambda: p.fetch_timing_json(ts)):
                with pytest.raises(capi.B200ddError) as e:
                    f()
                assert e.value.code == capi.FILTER_FAILED
            assert p.fetch_detection_stash() == stash
            continue
        assert not res["skipped"]
        ok, y_ref = O.wienerhopf_process(sc.x.astype(np.complex64).astype(np.complex128),
                                         sc.y.astype(np.complex64).astype(np.complex128), *clutter)
        ref, _, _ = O.ambiguity_process(sc.x.astype(np.complex64).astype(np.complex128),
                                        y_ref.astype(np.complex64).astype(np.complex128),
                                        O.ambiguity_geometry(*geom, True))
        e = relerr(m.cpu().numpy().astype(np.complex128), ref)
        assert ok and e[0] < 1e-5 and e[1] < 1e-5, (i, e)
        noise, mx = dh.set_metrics_device(m, gm.n_doppler_bins, gm.n_delay_bins)
        assert (noise, mx) == (res["noisePower"], res["maxPower"])
        d = dh.process_device_map(m, gm.n_doppler_bins, gm.n_delay_bins, p.delay, p.doppler, noise,
                                  capi.DET_INTERPOLATE)
        got = res["detections"]
        for u, v in ((got.delay, d.delay), (got.doppler, d.doppler), (got.snr, d.snr)):
            assert np.array_equal(u, v), i
        mj.render_device(m, noise, mx)
        assert p.fetch_map_json(ts) == mj.fetch(ts)
        p.fetch_detection_json(ts)
        n_cpi.append(json.loads(p.fetch_timing_json(ts))["nCpi"])
    assert n_cpi[1] == n_cpi[0] + 1  # the failed CPI in between did not step nCpi
    p.close()


def test_plan_world1_equals_the_pipeline():
    geom = "cfg2"
    g = GEOMS[geom]
    n = g["nSamples"]
    comm = Comm(0, 1, 0)
    for clutter in (None, g["clutter"]):
        a = _pipeline(geom, clutter=clutter)
        b = _pipeline(geom, clutter=clutter)
        amb = Ambiguity(g["delayMin"], g["delayMax"], g["dopplerMin"], g["dopplerMax"], g["fs"], n, True, device=0)
        sa = SpectrumAnalyser(n, 2000.0, device=0)
        plan = SingleCpiPlan(comm, amb, n, torch.device("cuda"), clutter=clutter,
                             whc_factory=lambda p, q, nn, c0, nc: WienerHopfChunk(p, q, nn, c0, nc, device=0),
                             spectrum=sa, pipeline=b)
        ma = _map_buf(a)
        s = torch.cuda.Stream()
        for i, (x, y) in enumerate(_scenes(geom)[:4]):
            a.submit_device(x, y, ma)
            torch.cuda.synchronize()
            pa, tma = _products(a, i)
            plan.x_own.copy_(x)
            plan.y_own.copy_(y)
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                plan.run(s)
            s.synchronize()
            pb, tmb = _products(b, i)
            if clutter is None:
                assert torch.equal(plan.map, ma), i
                assert pb == pa, i
            else:
                err = float((plan.map - ma).abs().max() / ma.abs().max())
                assert err < 1e-5, (i, err)
                assert dict(pb)["fetch"][:2] == dict(pa)["fetch"][:2]
                assert tmb["spectrum"] > 0 and tmb["clutter_filter"] > 0, tmb
            assert list(tmb) == list(tma)
        for p in (a, b):
            p.close()
    comm.close()


def test_refused_submit_map_enqueues_nothing():
    geom = "cfg2"
    g = GEOMS[geom]
    x, y = _scenes(geom)[0]
    sa = SpectrumAnalyser(g["nSamples"], 2000.0, device=0)
    part = torch.empty((1, sa.nSpectrum), dtype=torch.complex128, device="cuda")
    sa.fold_slice_device(x, 0, part[0])
    a = _pipeline(geom)
    m = _map_buf(a)
    a.submit_device(x, y, m)
    torch.cuda.synchronize()
    ref = _products(a, 0)[0]
    b = _pipeline(geom)
    st = _verdict(False)
    torch.cuda.synchronize()
    lib = b._lib
    h = b._h
    P = capi.ptr
    cases = [
        lambda: lib.b200dd_pipeline_submit_map(h, None, P(st), P(part), 1, None),
        lambda: lib.b200dd_pipeline_submit_map(h, P(m), None, P(part), 1, None),
        lambda: lib.b200dd_pipeline_submit_map(h, P(m), P(st), None, 0, None),
        lambda: lib.b200dd_pipeline_submit_map(h, P(m), P(st), P(part), 0, None),
        lambda: lib.b200dd_pipeline_stamp(h, 3, None),
    ]
    for c in cases:
        assert c() == capi.ERR_ARG
    nf = _pipeline(geom, clutter=None, spectrum=False)
    assert lib.b200dd_pipeline_submit_map(nf._h, P(m), P(st), None, 0, None) == capi.ERR_ARG
    assert lib.b200dd_pipeline_submit_map(nf._h, P(m), None, P(part), 1, None) == capi.ERR_ARG
    # a share-set member whose last CPI is not fetched
    s0, s1 = _pipeline(geom), _pipeline(geom)
    Pipeline.share_history([s0, s1])
    s0.submit_map(m, st.data_ptr(), part)
    assert lib.b200dd_pipeline_submit_map(s0._h, P(m), P(st), P(part), 1, None) == capi.ERR_ARG
    torch.cuda.synchronize()
    s0.fetch()
    # then a normal submit equals an untouched pipeline's
    b.submit_device(x, y, m)
    torch.cuda.synchronize()
    assert _products(b, 0)[0] == ref
    for p in (a, b, nf, s0, s1):
        p.close()
