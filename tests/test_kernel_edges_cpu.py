"""CPU: the edge-case tables of tests/edge_cases.py reach every default kernel instance, and the vectorised detection
restatements used on large maps are bit-identical to the oracle's loops."""
import ctypes as C

import numpy as np
import pytest

import edge_cases as E
from blah2_b200 import capi
from oracle import blah2_oracle as O


@pytest.mark.parametrize("row", E.CAF_ROWS, ids=E.row_id)
def test_row_geometry_and_plan(row):
    g = capi.caf_plan(*row["geom"])[0]
    og = O.ambiguity_geometry(*row["geom"])
    assert (g.n_delay_bins, g.n_doppler_bins, g.n_corr) == (row["n_del"], row["n_dop"], row["n_corr"])
    assert (og.nDelayBins, og.nDopplerBins, og.nCorr, og.nfft) == (g.n_delay_bins, g.n_doppler_bins, g.n_corr, g.nfft)
    assert (g.range_fft_len, g.doppler_fft_len) == (row["M"], row["M2"])
    assert 1 << E.plan_range_log2m(row["n_del"], row["n_corr"]) == row["M"]
    # every lag the map holds is inside the oracle's nfft-point correlation and inside a batch
    assert og.delayMax < og.nCorr and -og.delayMin < og.nCorr and og.nfft >= 2 * og.nCorr - 1
    # the segment plan covers a batch and leaves room for every lag
    assert g.range_segments * g.range_hop >= g.n_corr and g.range_hop + g.n_delay_bins - 1 <= g.range_fft_len


def test_rows_reach_every_default_kernel_instance():
    plans = [capi.caf_plan(*r["geom"])[0] for r in E.CAF_ROWS]
    ms = {int(g.range_fft_len) for g in plans}
    m2s = {int(g.doppler_fft_len) for g in plans}
    assert ms == {1 << l for l in range(8, 14)}
    assert m2s == {1 << l for l in range(8, 15)}
    kernels = {k for g in plans for k in E.default_kernels(int(g.range_fft_len), int(g.doppler_fft_len))}
    assert kernels == {f"caf_range_kernel<{l}>" for l in (8, 13)} | {f"caf_range_dit_kernel<{l}>" for l in range(9, 13)} \
        | {f"caf_doppler_kernel<{l}>" for l in (8, 13, 14)} | {f"caf_doppler_dit_kernel<{l}>" for l in range(9, 13)}
    # nDopplerBins on both sides of every Bluestein boundary: M2 doubles at nDop = 2^k + 1
    ndop = {int(g.n_doppler_bins) for g in plans}
    for k in range(7, 13):
        assert (1 << k) - 1 in ndop and (1 << k) + 1 in ndop, k
    assert 8191 in ndop


def test_range_switch_from_4096_to_8192_is_where_the_table_says():
    lo, hi = E.RANGE_SWITCH_4096_8192
    for n_del, M in ((lo, 4096), (hi, 8192)):
        assert 1 << E.plan_range_log2m(n_del, n_del + 100) == M
    # and nowhere else between the 3000-bin row and the 7168-bin row
    prev = None
    for n_del in range(3000, 7169, 7):
        M = 1 << E.plan_range_log2m(n_del, n_del + 100)
        assert M == (4096 if n_del <= lo else 8192), n_del
        prev = M
    assert prev == 8192


def test_widest_delay_window_advances_one_sample_per_segment():
    g = capi.caf_plan(*E._delay_row(8192, 8192)["geom"])[0]
    assert g.range_hop == 1 and g.range_segments == g.n_corr


@pytest.mark.parametrize("geom", E.CAF_REJECTED)
def test_planner_rejects_beyond_the_largest_instances(geom):
    lib = capi.load()
    p = capi.CafParams(*[int(v) for v in geom[:6]], int(geom[6]), -1)
    g = capi.CafGeometry()
    assert lib.b200dd_caf_plan(C.byref(p), C.byref(g), None, 0, None, 0) == capi.ERR_GEOMETRY


@pytest.fixture(scope="module")
def scene_map():
    return E.oracle_scene_map(seed=6)


@pytest.mark.parametrize("params", E.CFAR_PARAMS)
def test_vectorised_cfar_is_bit_identical_to_the_oracle(params, scene_map):
    g, m, noise = scene_map
    args = (params["pfa"], params["nGuard"], params["nTrain"], params["minDelay"], params["minDoppler"])
    ref = O.cfar_1d(m, g.delay, g.doppler, noise, *args)
    got = E.cfar_1d(m, g.delay, g.doppler, noise, *args)
    for a, b in zip(got, ref):
        assert a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("params", [E.CFAR_PARAMS[0], E.CFAR_PARAMS[4], E.CFAR_PARAMS[6]])
@pytest.mark.parametrize("n_centroid", [0, 2, 6, 70000])
def test_vectorised_centroid_is_bit_identical_to_the_oracle(params, n_centroid, scene_map):
    g, m, noise = scene_map
    det = O.cfar_1d(m, g.delay, g.doppler, noise, params["pfa"], params["nGuard"], params["nTrain"], params["minDelay"],
                    params["minDoppler"])
    assert det[0].shape[0] > 10
    res = g.doppler[1] - g.doppler[0]
    ref = O.centroid(*det, n_centroid, n_centroid, res)
    got = E.centroid(*det, n_centroid, n_centroid, res, chunk=97)
    for a, b in zip(got, ref):
        assert np.array_equal(a, b)


def test_vectorised_centroid_wraps_like_the_oracle():
    delay = np.array([2.0, 3.0, 4.0, 40.0, 41.0, 300.0, 65534.0, 1.0])
    dop = np.array([10.0, 11.0, 10.5, -20.0, -20.5, 0.0, 10.0, 10.0])
    snr = np.array([5.0, 9.0, 7.0, 3.0, 4.0, 1.0, 9.5, 9.0])
    for nd in (0, 1, 6, 65540):
        ref = O.centroid(delay, dop, snr, nd, 6, 1.0)
        got = E.centroid(delay, dop, snr, nd, 6, 1.0, chunk=3)
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), nd
