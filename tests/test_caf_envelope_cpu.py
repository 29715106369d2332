"""CPU: the rows of tests/caf_cases.py plan what they were written for and reach every default CAF kernel instance, the
scenes are exactly float32, the error model's bars are tight enough to matter, and a numpy FP32 restatement of the
kernels' segmented algorithm stays inside them (no device needed)."""
import math

import numpy as np
import pytest

import caf_cases as K
import edge_cases as E
from oracle import blah2_oracle as O


@pytest.mark.parametrize("row", K.ROWS, ids=K.row_id)
def test_row_plan(row):
    g = K.plan(row)
    og = O.ambiguity_geometry(*row["geom"])
    assert (g.n_delay_bins, g.n_doppler_bins, g.n_corr) == (og.nDelayBins, og.nDopplerBins, og.nCorr)
    env = row["env"]
    if "B200DD_CAF_LOG2M" in env:
        assert g.range_fft_len == 1 << int(env["B200DD_CAF_LOG2M"])
    if "B200DD_CAF_PARTS" in env:
        assert g.range_segments > 1 and g.range_parts == min(int(env["B200DD_CAF_PARTS"]), g.range_segments)
    assert g.range_segments * g.range_hop >= g.n_corr and g.range_hop + g.n_delay_bins - 1 <= g.range_fft_len
    # every lag inside a batch and inside the oracle's nfft-point correlation
    assert og.delayMax < og.nCorr and -og.delayMin < og.nCorr and og.nfft >= 2 * og.nCorr - 1


def test_rows_reach_every_default_kernel_instance():
    plans = [K.plan(r) for r in K.ROWS if not r["env"]]
    kernels = {k for g in plans for k in E.default_kernels(int(g.range_fft_len), int(g.doppler_fft_len))}
    assert kernels == {f"caf_range_kernel<{l}>" for l in (8, 13)} | {f"caf_range_dit_kernel<{l}>" for l in range(9, 13)} \
        | {f"caf_doppler_kernel<{l}>" for l in (8, 13, 14)} | {f"caf_doppler_dit_kernel<{l}>" for l in range(9, 13)}
    forced = {int(K.plan(r).range_fft_len) for r in K.ROWS if "B200DD_CAF_LOG2M" in r["env"]}
    assert forced == {1 << l for l in range(8, 14)}
    # a hop of one sample (one x sample per segment) and many segments per part
    assert any(int(g.range_hop) == 1 and -(-int(g.range_segments) // int(g.range_parts)) > 500 for g in plans)


def test_off_centre_rows_rotate_past_a_thousand_radians():
    phases = []
    for r in K.ROWS:
        og = O.ambiguity_geometry(*r["geom"])
        if og.dopplerMiddle != 0 and og.n >= 10 ** 6:
            phases.append(2 * math.pi * abs(og.dopplerMiddle) * og.n_used / og.fs)
    assert len(phases) >= 2 and min(phases) > 1e3


@pytest.mark.parametrize("case", [c for c in K.cases() if c[0]["id"] not in K.FULL_SIZE], ids=K.case_id)
def test_scene_is_float32_and_the_bar_is_tight(case):
    row, scene = case
    g = K.plan(row)
    x, y = K.make_input(row, scene)
    og = O.ambiguity_geometry(*row["geom"])
    assert x.dtype == y.dtype == np.complex64 and x.shape[0] >= og.n_used and np.all(np.isfinite(x)) and np.all(np.isfinite(y))
    assert np.array_equal(x.astype(np.complex128).astype(np.complex64), x)
    if scene in ("white", "narrowband", "fc32"):      # fractional samples: the first butterflies round
        assert np.any(x.real != np.round(x.real)) and np.any(y.real != np.round(y.real))
    R, ref = K.reference(row, x, y)
    rb, mb = K.error_model(row, g, x, y, R)
    assert rb.shape == (og.nDopplerBins,) and mb.shape == (og.nDopplerBins, og.nDelayBins)
    assert np.all(rb > 0) and np.all(mb > 0)
    mx = float(np.max(np.abs(ref)))
    # at least 6x tighter than the 1e-5 of the largest cell that the parity tests use where a direct path or a tone
    # dominates the map (its fixed-gain leakage alone is ~7u of the peak); where nothing does (white inputs, the
    # filtered scene on short CPIs) the largest cell is only ~4 rms above the rest and the FP32 error of the algorithm
    # itself reaches ~6u of it: there at least 2.5x (the hop-1 row, whose 638-step accumulations dominate, is the worst)
    assert np.max(mb) <= (4e-6 if scene in ("white", "filtered") else 1.5e-6) * mx, float(np.max(mb) / mx)
    if scene in ("direct", "filtered"):
        assert np.median(K.db_bar(ref, mb)) < 0.005


@pytest.mark.parametrize("case", [c for c in K.cases() if K.affordable(c[0], K.plan(c[0]))], ids=K.case_id)
def test_fp32_restatement_stays_inside_the_model(case):
    row, scene = case
    g = K.plan(row)
    x, y = K.make_input(row, scene)
    R, ref = K.reference(row, x, y)
    rb, mb = K.error_model(row, g, x, y, R)
    Rf, mf = K.restate_fp32(row, g, x, y)
    er = np.max(np.abs(Rf - R), axis=1) / rb
    em = np.abs(mf - ref) / mb
    assert np.max(er) <= 1.0, (int(np.argmax(er)), float(np.max(er)))
    assert np.max(em) <= 1.0, (np.unravel_index(int(np.argmax(em)), em.shape), float(np.max(em)))
