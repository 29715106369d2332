"""GPU: the spectrum stage bin by bin at every row of tests/spectrum_cases.py, on each of its entry points, against
numpy's FP64 FFT of the same samples (oracle.blah2_oracle.spectrum_process).

Entry points: process_device on float2 starting 16-byte aligned (the two-column fold when the bin count is even),
the same on float2 starting 8-byte aligned (the one-column fold), process_device on complex128 (the _f64 entry) and
process (the host path).  Every device buffer is guard-banded with NaN, and the samples in [nfft, n), which the
reference never reads, are NaN too.

The input is what blah2's reference channel looks like: float32-representable, non-integer noise (unit variance per
component) under a tone 114 dB and a DC offset 103 dB above it.  The tone sits on a kept bin; the DC usually does
not, so it cancels in the fold.  The IQ-data document prints 10 log10 |s| of every bin, and a check relative to the
largest bin at 1e-11 lets a bin 100 dB down be wrong by whole dB.  Here every bin is checked against the error
model of the kernels (u = 2^-53, g = the folded vector the DFT transforms, computed here in numpy):

    |s_m - ref_m| <= u ( sum_r |g_r| (j_r + 1)                     running-product drift
                         + 2 sqrt(A_dft) ||g||_1                   DFT additions
                         + 2 sqrt(A_fold) ||x[:nfft]||_1           fold additions
                         + 4 sqrt(log2 nfft) ||x[:nfft]||_2 )      numpy's own FFT

j_r is the number of running-product steps since the phase of term r was seeded from the table (at most
DFT_RESEED - 1 = 63); a step's error is at most u and is common to every term of a chain, so it adds up coherently.
A_fold counts the additions a sample goes through (the rows of its chunk, the chunks of its warp, the warps of the
chunk reduction), A_dft those of a DFT term (its chain, 4 ILP lanes, 32 slices); independent roundings add up with
the square root of their count.  The strong components cancel in the fold (the DC) or fill one bin (the tone), and
the rounding errors of both spread over every bin: the measured errors on bins far from the tone reach 2400 u
||x||_2 on the 2e7-sample row, so the bound is in l1 norms.  On these inputs it is 1e-14 of max |s| or less: at
least 1000x tighter than the 1e-11 bar of tests/test_spectrum_gpu.py, which it asserts on every row.

Measured worst ratio |s_m - ref_m| / bar over all rows, bins and the four entry points on an H100: 0.30.  A DFT that does not re-seed its running products (512-step chains at 65536 bins)
exceeds the bar by 18 - 24 % on the 65536-bin rows; phase tables rounded to float exceed it 10^6-fold.
"""
import math

import numpy as np
import pytest
import torch

import spectrum_cases as S
from blah2_b200.process import SpectrumAnalyser
from guarded import Guarded
from oracle import blah2_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
ENTRY_POINTS = ("float2_aligned", "float2_misaligned", "f64", "host")


def make_input(r, seed):
    """n samples: float32-representable noise + tone + DC in [0, nfft), NaN in [nfft, n)."""
    n, ns, dec, nfft = r["n"], r["n_spectrum"], r["dec"], r["nfft"]
    rng = np.random.default_rng(seed)
    k0 = nfft // 2 + 1
    m0 = ns // 3
    k_tone = (m0 * dec + k0) % nfft
    ph = (np.arange(nfft, dtype=np.int64) * k_tone) % nfft
    x = rng.standard_normal(nfft) + 1j * rng.standard_normal(nfft)
    x += 7e5 * np.exp(2j * np.pi * ph / nfft) + 2e5 * (0.6 - 0.8j)
    out = np.full(n, complex(np.nan, np.nan), dtype=np.complex64)
    out[:nfft] = x.astype(np.complex64)
    return out, m0


def run_entry_points(r, x):
    """{entry point: spectrum} with every guard checked and every device entry point run twice (bit-identical)."""
    sa = SpectrumAnalyser(r["n"], r["bw"])
    assert (sa.decimation, sa.nSpectrum, sa.nfft) == (r["dec"], r["n_spectrum"], r["nfft"])
    ns, n = sa.nSpectrum, r["n"]
    out = {}
    for name, off, dt in (("float2_aligned", 0, torch.complex64), ("float2_misaligned", 1, torch.complex64),
                          ("f64", 0, torch.complex128)):
        bx = Guarded(n, off, x, dtype=dt)
        runs = []
        for _ in range(2):
            bo = Guarded(ns, 1, dtype=torch.complex128)
            torch.cuda.synchronize()
            sa.process_device(bx.view, d_spectrum=bo.view)
            torch.cuda.synchronize()
            assert bx.intact() and bo.intact(), name
            runs.append(bo.numpy())
        assert np.array_equal(runs[0], runs[1]), f"{name}: a repeated run differs"
        out[name] = runs[0]
    host = [sa.process(x.astype(np.complex128))[0] for _ in range(2)]
    assert np.array_equal(host[0], host[1]), "host: a repeated run differs"
    out["host"] = host[0]
    geom = sa.geometry
    sa.close()
    return out, geom


def folded(x, r):
    """g[r] = exp(-2 pi i k0 r / nfft) sum_q x[q nSpectrum + r] exp(-2 pi i k0 q / decimation), in FP64."""
    nfft, ns, dec = r["nfft"], r["n_spectrum"], r["dec"]
    k0 = nfft // 2 + 1
    t = np.exp(-2j * np.pi * ((np.arange(nfft, dtype=np.int64) * k0) % nfft) / nfft)
    return (x[:nfft].astype(np.complex128) * t).reshape(dec, ns).sum(axis=0)


def error_bar(r, geom, x):
    """The bound of the module docstring, one number for every bin of the row."""
    ns, nfft = r["n_spectrum"], r["nfft"]
    steps = np.arange(ns) // 128                 # a chain steps 32 slices x 4 ILP lanes = 128 bins
    if ns > S.DFT_RESEED_FROM:
        steps %= 64                              # re-seeded every DFT_RESEED = 64 steps
    rows, chunks = int(geom.fold_rows_per_chunk), int(geom.fold_chunks)
    a_fold = min(rows, r["dec"]) + math.ceil(chunks / 32) + min(chunks, 32)
    a_dft = math.ceil(ns / 128) + 4 + 32
    xs = x[:nfft].astype(np.complex128)
    ag = np.abs(folded(x, r))
    return U * (float(np.sum(ag * (steps + 1))) + 2 * math.sqrt(a_dft) * float(ag.sum())
                + 2 * math.sqrt(a_fold) * float(np.sum(np.abs(xs)))
                + 4 * math.sqrt(max(1.0, math.log2(nfft))) * float(np.linalg.norm(xs)))


@pytest.mark.parametrize("r", S.ROWS, ids=S.row_id)
def test_spectrum_per_bin_on_every_entry_point(r):
    x, _ = make_input(r, seed=r["n_spectrum"] * 31 + r["dec"])
    ref, _ = O.spectrum_process(x.astype(np.complex128), r["n"], r["bw"])
    assert np.all(np.isfinite(ref))
    out, geom = run_entry_points(r, x)
    bar = error_bar(r, geom, x)
    smax = float(np.max(np.abs(ref)))
    assert bar <= 1e-13 * smax     # at least 100x tighter than 1e-11 of the largest bin
    for name in ENTRY_POINTS:
        s = out[name]
        assert s.shape == ref.shape and np.all(np.isfinite(s)), name
        err = np.abs(s - ref)
        worst = int(np.argmax(err))
        assert err[worst] <= bar, (name, worst, float(err[worst] / bar), float(np.abs(ref[worst])))
    # the two float2 folds are the same sums grouped differently; the one-column fold on float2 and on its
    # widening to complex128 is the same arithmetic, and so are the _f64 entry point and the host path
    a, b = out["float2_aligned"], out["float2_misaligned"]
    assert np.max(np.abs(a - b)) <= 1e-13 * smax
    if r["n_spectrum"] % 2:
        assert np.array_equal(a, b)
    assert np.array_equal(out["float2_misaligned"], out["f64"])
    assert np.array_equal(out["f64"], out["host"])
