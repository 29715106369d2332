"""GPU: the delay-Doppler map cell by cell, and the range matrix row by row, against the FP32 error model of
tests/caf_cases.py at every row and scene of that table, on every CAF entry point; the map document and the CFAR
decisions of the device map against those of the FP64 map.

Entry points, and the arithmetic they share:
  host        Ambiguity.process: complex128 in, converted (and pre-rotated) in double on the device, rounded to float
  aligned     process_device on float2 starting 16-byte aligned, in NaN-guarded buffers
  misaligned  the same starting 8-byte aligned
  tiles       range_device on all batches + doppler_device on 2 and on 3 column tiles + place_tiles (symmetric windows)
  pipeline    Pipeline.submit_device without clutter filter or detection
All of them run the same kernels on the same float samples: the pre-rotation (dopplerMiddle != 0) is the same double
arithmetic on the same values in caf_convert_kernel and caf_prerotate_kernel, the TMA-staged loads are exact, the tile
path sums the parts in the order the Doppler kernel does, and the pipeline calls process_device.  So every entry point
must give the one map bit for bit, and a repeated run the same bits.

Map document: the device map's and the FP64 map's documents (same noisePower and maxPower) may differ in a cell only
where the FP64 value lies within the dB-converted bar of a hundredths rounding boundary.  CFAR (direct-path and
filtered scenes): a decision may differ only where |sq - thr| lies within the bar carried through |z|^2 and the
training mean.
"""
import json

import numpy as np
import pytest
import torch

import caf_cases as K
import edge_cases as E
from blah2_b200.process import Ambiguity, MapJson, Pipeline
from blah2_b200.shard import block_range
from guarded import Guarded
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

CFAR = E.CFAR_PARAMS[0]


def _sync():
    torch.cuda.synchronize()


def _device_runs(amb, x, y, cells):
    """{entry point: map [nDop, nDel] complex64}; guards checked, every device entry point run twice."""
    g = amb.geometry
    shape = (g.n_doppler_bins, g.n_delay_bins)
    n = x.shape[0]
    out = {}
    for name, off in (("aligned", 0), ("misaligned", 1)):
        bx, by = Guarded(n, off, x), Guarded(n, off, y)
        runs = []
        for _ in range(2):
            bm = Guarded(cells, 1)
            _sync()
            amb.process_device(bx.view, by.view, bm.view)
            _sync()
            assert bx.intact() and by.intact() and bm.intact(), name
            runs.append(bm.numpy().reshape(shape))
        assert np.array_equal(runs[0], runs[1]), f"{name}: a repeated run differs"
        out[name] = runs[0]
    if g.doppler_middle == 0.0:
        dx = torch.from_numpy(x[: g.n_used]).cuda()
        dy = torch.from_numpy(y[: g.n_used]).cuda()
        for nt in (2, 3):
            R = Guarded(cells, 1)
            amb.range_device(dx, dy, 0, g.n_doppler_bins, R.view)
            tiles = Guarded(cells, 0)
            off = 0
            for t in range(nt):
                c0, nc = block_range(g.n_delay_bins, t, nt)
                amb.doppler_device(R.view, c0, nc, tiles.view[off:off + g.n_doppler_bins * nc])
                off += g.n_doppler_bins * nc
            m = Guarded(cells, 1)
            amb.place_tiles(tiles.view, nt, m.view)
            _sync()
            assert R.intact() and tiles.intact() and m.intact(), nt
            out[f"tiles{nt}"] = m.numpy().reshape(shape)
    return out


def _pipeline_map(row, x, y, cells):
    geom = row["geom"]
    pipe = Pipeline(*geom[:6], roundHamming=geom[6])
    dx, dy = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    bm = Guarded(cells, 1)
    s = torch.cuda.Stream()
    _sync()
    with torch.cuda.stream(s):
        pipe.submit_device(dx, dy, bm.view, s.cuda_stream)
        pipe.fetch(s.cuda_stream)
    s.synchronize()
    assert bm.intact()
    g = pipe.geometry
    out = bm.numpy().reshape(g.n_doppler_bins, g.n_delay_bins)
    pipe.close()
    return out


def _doc_cells(doc):
    return np.asarray(json.loads(doc)["data"], dtype=np.float64)


def _check_document(amb, geom, m, ref, mb):
    """Number of cells whose text differs; each one must be explained by the bar."""
    noise, mx = O.set_metrics(ref)
    mj = MapJson(amb.delay, amb.doppler, geom[4])
    mj.render_device(torch.from_numpy(m).cuda(), noise, mx)
    dev = _doc_cells(mj.fetch(1700000000000))
    host = _doc_cells(mj.render_host(ref, noise, mx, 1700000000000))
    mj.close()
    assert dev.shape == host.shape
    diff = dev != host
    if not diff.any():
        return 0
    v = 10.0 * np.log10(np.abs(ref)) - noise                 # the FP64 value of every cell
    if v.shape != diff.shape:
        v = v.T
    dbb = K.db_bar(ref, mb)
    if dbb.shape != diff.shape:
        dbb = dbb.T
    to_boundary = np.abs(v * 100.0 - np.round(v * 100.0)) / 100.0     # the text truncates to hundredths
    bad = diff & ((to_boundary > dbb + 1e-12) | (np.abs(dev - host) > 0.0100001))
    assert not bad.any(), [(tuple(int(i) for i in c), float(dev[tuple(c)]), float(host[tuple(c)]), float(v[tuple(c)]))
                           for c in np.argwhere(bad)[:5]]
    return int(diff.sum())


def _check_cfar(amb, m, ref, mb):
    """Number of flipped decisions; each one must be explained by the bar."""
    noise, _ = O.set_metrics(ref)
    args = (CFAR["pfa"], CFAR["nGuard"], CFAR["nTrain"], CFAR["minDelay"], CFAR["minDoppler"])
    det_ref, margin, cells, alpha = K.cfar_margins(ref, amb.delay, amb.doppler, *args)
    det_dev, _, _, _ = K.cfar_margins(m.astype(np.complex128), amb.delay, amb.doppler, *args)
    slack = K.cfar_slack(ref, mb, CFAR["nGuard"], CFAR["nTrain"], alpha, cells)
    flip = det_ref != det_dev
    bad = flip & (np.abs(margin) > slack)
    assert not bad.any(), np.argwhere(bad)[:5].tolist()
    # the decisions of the device map, as the detection restatement lists them, are the set tested here
    d = E.cfar_1d(m.astype(np.complex128), amb.delay, amb.doppler, noise, *args)
    assert d[0].shape[0] == int(det_dev.sum())
    return int(flip.sum())


# Known misses of the model, measured on an H100 (DESIGN s2): the map cell at the ratio given exceeds its bar.  Strict:
# a fix that brings them inside makes these fail until the mark goes.
KNOWN_MISSES = {
    "edge-nDop31-nDel8192-narrowband": "zero-Doppler cell at delay bin 8179: 1.32 x the bar.  Hop 1: 638 cross-spectra "
                                       "of a tone accumulated per part, whose roundings are not independent",
    "offcentre-down-filtered": "cell (659, 118): 1.05 x the bar",
}


def _params():
    out = []
    for c in K.cases():
        why = KNOWN_MISSES.get(K.case_id(c))
        out.append(pytest.param(c, id=K.case_id(c),
                                marks=[pytest.mark.xfail(strict=True, reason=why)] if why else []))
    return out


@pytest.mark.parametrize("case", _params())
def test_caf_within_the_fp32_error_model(case, monkeypatch):
    row, scene = case
    if row["id"] in K.FULL_SIZE:
        monkeypatch.setenv("BLAH2_ORACLE_WORKERS", "-1")
    for k, v in row["env"].items():
        monkeypatch.setenv(k, v)
    geom = row["geom"]
    g = K.plan(row)
    x, y = K.make_input(row, scene)
    R, ref = K.reference(row, x, y)
    rb, mb = K.error_model(row, g, x, y, R)
    kern = E.default_kernels(int(g.range_fft_len), int(g.doppler_fft_len))
    tag = f"{row['id']} {scene} {kern[0]} + {kern[1]}"

    amb = Ambiguity(*geom)
    ag = amb.geometry
    assert (ag.range_fft_len, ag.range_hop, ag.range_segments, ag.range_parts, ag.doppler_fft_len) == \
        (g.range_fft_len, g.range_hop, g.range_segments, g.range_parts, g.doppler_fft_len)
    x128, y128 = x.astype(np.complex128), y.astype(np.complex128)
    host = amb.process(x128, y128).data
    Rd = amb.debug_range_matrix()
    assert np.array_equal(amb.process(x128, y128).data, host), f"{tag}: a repeated host run differs"
    assert np.all(np.isfinite(host)) and np.all(np.isfinite(Rd))

    # range stage, row by row
    er = np.max(np.abs(Rd.astype(np.complex128) - R), axis=1) / rb
    i = int(np.argmax(er))
    assert er[i] <= 1.0, f"{tag}: range row {i}: error / bar = {er[i]:.3g}"
    # map, cell by cell against its bar
    em = np.abs(host - ref) / mb
    k, j = np.unravel_index(int(np.argmax(em)), em.shape)
    assert em[k, j] <= 1.0, f"{tag}: map cell (doppler {k}, delay {j}): error / bar = {em[k, j]:.3g}"
    ratios = (float(er[i]), float(em[k, j]))

    cells = ag.n_doppler_bins * ag.n_delay_bins
    maps = _device_runs(amb, x, y, cells)
    maps["pipeline"] = _pipeline_map(row, x, y, cells)
    m32 = host.astype(np.complex64)
    assert np.array_equal(m32.astype(np.complex128), host)
    for name, m in maps.items():
        assert np.array_equal(m, m32), f"{tag}: {name} differs from the host path"

    flips = ndiff = "-"
    if scene in ("direct", "filtered"):
        ndiff = _check_document(amb, geom, m32, ref, mb)
        flips = _check_cfar(amb, m32, ref, mb)
    amb.close()
    print(f"\nCAF-ENVELOPE {tag}: range {ratios[0]:.3f} map {ratios[1]:.3f} bar/max {np.max(mb) / np.max(np.abs(ref)):.2e} "
          f"doc-cells-differing {ndiff} cfar-flips {flips}")
