"""Ill-conditioned clutter-filter scenes and an exact truth, shared by tests/test_wh_conditioning_cpu.py and
tests/test_wh_conditioning_gpu.py.

A white reference channel gives a Toeplitz matrix A with cond(A) ~ 1, where every FP64 solver is accurate to a few
ulp.  Real references are not white: an FM broadcast fills ~10 % of blah2's 2 MS/s band, DVB-T leaves guard bands,
SDRs add a DC offset and pilots add strong tones.  The solve multiplies its rounding errors by cond(A) (up to ~1e12
here), so a kernel's accuracy there is compared with what the oracle's LAPACK Cholesky achieves on the same system,
and both are measured against an exact truth:

* The inputs are integers (int16 scale, sigma ~ 1500, or int8 scale, sigma ~ 30) and N <= 2^18.  The correlations
  a[k] and b[k] are plain sums of products (the reference's 1/N cancels its unnormalised IFFT), so they are integers
  below 2^50.  The oracle's FP64 FFT correlations are within far less than 0.5 of them; rounding gives
  the exact values (exact_correlations).
* The system A w = b has integer entries.  Iterative refinement from LAPACK's cho_solve, with every residual
  computed exactly (10-bit integer limbs, whose FFT convolutions stay far enough below 2^53 to round to the exact
  integers), converges to w to ~2^-61 of max|w| (exact_weights).
* y' = y - (xs * w)[:N] is computed the same way: integer limbs of w, FFT convolutions of integers rounded to the
  exact integers they are (exact_output).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import scipy.linalg as sla

from oracle import blah2_oracle as O

# (name, occupied fraction of the band, DC offset / sigma, tone power over the band's power in dB)
REFERENCES = [
    ("white", 1.0, 0.0, None),
    ("occ50", 0.5, 0.0, None),
    ("occ10", 0.1, 0.0, None),
    ("occ2", 0.02, 0.0, None),
    ("occ10_dc", 0.1, 2.0, None),
    ("occ10_tone", 0.1, 0.0, 20.0),
]
# integer sample scales: (name, sigma of the reference, receiver noise sigma, clip level)
SCALES = {"int16": (1500.0, 20.0, 32767), "int8": (30.0, 0.4, 127)}

FS = 2000000
MOVER = (25, 300.0, -50.0)       # (delay bin, Doppler Hz, dB): make_scene's Target


def _round_clip(v, lim):
    return np.clip(np.round(v.real), -lim, lim) + 1j * np.clip(np.round(v.imag), -lim, lim)


@dataclass
class Scene:
    name: str
    x: np.ndarray       # complex128, integer valued
    y: np.ndarray


def make_reference(n, occupied, dc, tone_db, sigma, lim, rng):
    """Complex Gaussian band-limited to the `occupied` fraction of the band around 0 Hz by zeroing FFT bins, plus a
    DC offset (dc sigma), then rounded to integers.  With a tone, the tone takes 0.45 of the clip level and the band
    sits tone_db below it."""
    u = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / math.sqrt(2.0)
    if occupied < 1.0:
        f = np.fft.fftfreq(n)
        U = np.fft.fft(u)
        U[np.abs(f) >= occupied / 2.0] = 0.0
        u = np.fft.ifft(U)
        u /= math.sqrt(np.mean(np.abs(u) ** 2))
    if tone_db is not None:
        amp = 0.3 * lim
        sigma = amp * 10.0 ** (-tone_db / 20.0)
    x = sigma * u
    if dc:
        x = x + dc * sigma * np.exp(2j * np.pi * rng.uniform())
    if tone_db is not None:
        f0 = occupied * rng.uniform(0.1, 0.4)
        x = x + amp * np.exp(2j * np.pi * (f0 * np.arange(n) + rng.uniform()))
    return _round_clip(x, lim)


def make_case_scene(ref_name, scale, n, seed):
    """make_scene's surveillance channel on a conditioned reference: direct path at -6 dB, static clutter taps at
    delays 1-15 falling from -10 to -40 dB, the -50 dB mover MOVER and receiver noise, rounded to integers."""
    _, occ, dc, tone = {r[0]: r for r in REFERENCES}[ref_name]
    sigma, sigma_noise, lim = SCALES[scale]
    rng = np.random.default_rng(seed)
    x = make_reference(n, occ, dc, tone, sigma, lim, rng)
    y = 0.5 * x
    for d in range(1, 16):
        g_db = -10.0 - 30.0 * (d - 1) / 14.0
        y[d:] += 10.0 ** (g_db / 20.0) * np.exp(1j * rng.uniform(0, 2 * np.pi)) * x[:-d]
    d, fd, g_db = MOVER
    mover = np.zeros(n, dtype=np.complex128)
    mover[d:] = x[:n - d]
    y = y + 10.0 ** (g_db / 20.0) * mover * np.exp(2j * np.pi * fd * np.arange(n) / FS)
    y = y + (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * (sigma_noise / math.sqrt(2.0))
    return Scene(f"{ref_name}_{scale}", x, _round_clip(y, lim))


def scene_seed(ref_name, scale):
    return 100 * [r[0] for r in REFERENCES].index(ref_name) + list(SCALES).index(scale) + 11


# ------------------------------------------------------------------------------------------------ exact truth
def shifted_reference(x, delayMin):
    """xs of WienerHopf.cpp:65-69 (oracle.wienerhopf_weights), with the uint32 wrap for delayMin > 0."""
    n = x.shape[0]
    t = (np.arange(n, dtype=np.int64) - int(delayMin)) % (1 << 32)
    return x[((t % n) + n) % n]


def exact_correlations(x, y, delayMin, delayMax):
    """(a, b, max distance to the nearest integer): a[k] and b[k] of oracle.wienerhopf_weights, computed the same
    way (FP64 FFTs, the delayMin wrap) and rounded to the integers they are."""
    nb = delayMax - delayMin
    xs = shifted_reference(x, delayMin)
    X, Y = np.fft.fft(xs), np.fft.fft(y)
    na = np.conj(np.fft.ifft(X * np.conj(X))[:nb])
    nbv = np.fft.ifft(Y * np.conj(X))[:nb]
    ra, rb = _round_c(na), _round_c(nbv)
    dist = max(np.max(np.abs(na - ra)), np.max(np.abs(nbv - rb)))
    return ra, rb, float(dist)


def _round_c(v):
    return np.round(v.real) + 1j * np.round(v.imag)


def correlation_lag_int64(x, y, delayMin, k):
    """a[k] and b[k] at one lag as int64 dot products (the circular correlations of WienerHopf.cpp:76-108)."""
    xs = shifted_reference(x, delayMin)
    xr, xi = xs.real.astype(np.int64), xs.imag.astype(np.int64)
    yr, yi = y.real.astype(np.int64), y.imag.astype(np.int64)
    sr, si = np.roll(xr, -k), np.roll(xi, -k)       # xs[(i + k) mod N]
    # a[k] = conj(sum xs[i+k] conj(xs[i])), b[k] = sum y[i+k] conj(xs[i])
    ar = int(np.dot(sr, xr) + np.dot(si, xi))
    ai = -int(np.dot(si, xr) - np.dot(sr, xi))
    tr, ti = np.roll(yr, -k), np.roll(yi, -k)
    br = int(np.dot(tr, xr) + np.dot(ti, xi))
    bi = int(np.dot(ti, xr) - np.dot(tr, xi))
    return complex(ar, ai), complex(br, bi)


def toeplitz_matrix(a):
    """The matrix the reference builds (WienerHopf.cpp:85-97): A(i, j) = a[j - i] for j >= i, conj(a[i - j]) below."""
    return sla.toeplitz(np.conj(a), a)


LIMB = 10             # bits per limb: every convolution below ~2^40, so its FP64 FFT is off by far less than 0.5
W_TOP = 61            # fixed point: max |w| ~ 2^61 units


def _limbs(v, count):
    """Complex integer vector v (integer-valued float real and imaginary parts, |.| < 2^(LIMB count)) as `count`
    complex limbs, v = sum_q L_q 2^(LIMB q), every part of every limb below 2^LIMB in magnitude."""
    out = []
    for part in (np.rint(v.real).astype(np.int64), np.rint(v.imag).astype(np.int64)):
        r, ls = part.copy(), []
        for _ in range(count - 1):
            lo = r & ((1 << LIMB) - 1)
            ls.append(lo)
            r = (r - lo) >> LIMB
        assert np.all(np.abs(r) < (1 << LIMB)), "value out of the limbs' range"
        ls.append(r)
        out.append(ls)
    return [lr.astype(np.float64) + 1j * li.astype(np.float64) for lr, li in zip(*out)]


def _exact_conv_sum(pairs, L, n0, n):
    """Linear convolution sum_k (u_k * v_k)[n0 : n0 + n] of complex integer sequences by FP64 FFTs, rounded to the
    integers it is (the transforms' error is asserted far below 0.5)."""
    acc = np.zeros(L, dtype=np.complex128)
    for U, V in pairs:
        acc += U * V
    c = np.fft.ifft(acc)[n0:n0 + n]
    cr, ci = np.round(c.real), np.round(c.imag)
    assert max(np.max(np.abs(c.real - cr)), np.max(np.abs(c.imag - ci))) < 0.05, "FFT convolution not exact"
    return cr.astype(np.int64), ci.astype(np.int64)


def _big(v):
    return np.array([int(t) for t in v], dtype=object)


def _to_float(v, S):
    return np.ldexp(np.array([float(t) for t in v]), -S)


def _fixed_point(w):
    """(W, S): w = W 2^-S with max |W| ~ 2^W_TOP, W a complex integer vector."""
    S = W_TOP - int(math.ceil(math.log2(np.max(np.abs(w)))))
    assert S >= 0
    return np.rint(np.ldexp(w.real, S)) + 1j * np.rint(np.ldexp(w.imag, S)), S


def _toeplitz_matvec_exact(Na, W):
    """toeplitz_matrix(Na) W for complex integer vectors Na (|.| < 2^50) and W (|.| < 2^63), exactly, as Python
    integers (real, imag).  (A W)_i = sum_j t[j - i] W_j with t[s] = Na[s], conj(Na[-s]) below: row i of the product
    is element n - 1 + i of the convolution of u[m] = t[n - 1 - m] with W."""
    n = Na.shape[0]
    t = np.concatenate([np.conj(Na[:0:-1]), Na])           # t[s], s = -(n - 1) .. n - 1
    u = t[::-1]
    L = 1 << int(math.ceil(math.log2(3 * n)))
    Uf = [np.fft.fft(l, n=L) for l in _limbs(u, 5)]
    Wf = [np.fft.fft(l, n=L) for l in _limbs(W, 7)]
    rr = np.zeros(n, dtype=object)
    ri = np.zeros(n, dtype=object)
    for g in range(5 + 7 - 1):
        pairs = [(Uf[p], Wf[g - p]) for p in range(5) if 0 <= g - p < 7]
        cr, ci = _exact_conv_sum(pairs, L, n - 1, n)
        rr += _big(cr) * (1 << (LIMB * g))
        ri += _big(ci) * (1 << (LIMB * g))
    return rr, ri


@dataclass
class Truth:
    w: np.ndarray       # the exact solution, rounded to complex128
    iterations: int


def exact_weights(Na, Nb, cf=None, max_iter=30):
    """w with A w = b to ~2^-61 max|w|: LAPACK's Cholesky solve, refined with exact residuals in fixed point
    (w = W 2^-S, W integer), until the correction is below 2^-53 max|w|."""
    assert np.max(np.abs(Na)) < 2.0 ** 50
    cf = cf or sla.cho_factor(toeplitz_matrix(Na), lower=False, check_finite=True)
    W, S = _fixed_point(sla.cho_solve(cf, Nb))
    br, bi = _big(Nb.real) * (1 << S), _big(Nb.imag) * (1 << S)
    for it in range(1, max_iter + 1):
        mr, mi = _toeplitz_matvec_exact(Na, W)
        d = sla.cho_solve(cf, _to_float(br - mr, 0) + 1j * _to_float(bi - mi, 0))   # correction in units of 2^-S
        W = W + (np.rint(d.real) + 1j * np.rint(d.imag))
        if np.max(np.abs(d)) <= 2.0 ** (W_TOP - 53):
            return Truth(np.ldexp(W.real, -S) + 1j * np.ldexp(W.imag, -S), it)
    raise AssertionError(f"iterative refinement did not converge in {max_iter} steps")


def cond_estimate(A, cf):
    """LAPACK's 1-norm condition estimate of a Hermitian positive-definite A from its Cholesky factor (zpocon): the
    order of magnitude the case ids report."""
    rcond, info = sla.lapack.zpocon(cf[0], np.max(np.sum(np.abs(A), axis=0)), uplo="L" if cf[1] else "U")
    assert info == 0
    return float(1.0 / rcond)


def exact_output(x, y, delayMin, w):
    """y' = y - (xs * w)[:N] (WienerHopf.cpp:125-160, a linear convolution), w taken exactly as its fixed-point
    value: FFT convolutions of xs with w's integer limbs, each rounded to the integers it is, summed exactly."""
    n, nb = x.shape[0], w.shape[0]
    W, S = _fixed_point(w)
    L = O.next_hamming(n + nb)
    X = np.fft.fft(shifted_reference(x, delayMin), n=L)
    acc_r, acc_i = _big(y.real) * (1 << S), _big(y.imag) * (1 << S)
    for q, l in enumerate(_limbs(W, 7)):
        cr, ci = _exact_conv_sum([(X, np.fft.fft(l, n=L))], L, 0, n)
        acc_r -= _big(cr) * (1 << (LIMB * q))
        acc_i -= _big(ci) * (1 << (LIMB * q))
    return _to_float(acc_r, S) + 1j * _to_float(acc_i, S)


def mp_levinson(Na, Nb, dps=50):
    """w of toeplitz_matrix(Na) w = Nb by the Levinson-Durbin recursion in mpmath at `dps` digits."""
    import mpmath as mp
    with mp.workdps(dps):
        return _mp_levinson(mp, Na, Nb)


def _mp_levinson(mp, Na, Nb):
    n = len(Na)
    col = [mp.mpc(complex(np.conj(v))) for v in Na]      # A(i, 0) = conj(a[i])
    row = [mp.mpc(complex(v)) for v in Na]               # A(0, j) = a[j]
    b = [mp.mpc(complex(v)) for v in Nb]
    f, g = [1 / row[0]], [1 / row[0]]                    # forward / backward vectors of the leading minors
    x = [b[0] / row[0]]
    for k in range(1, n):
        ef = sum(col[k - i] * f[i] for i in range(k))          # row k of A times [f, 0]
        eb = sum(row[i + 1] * g[i] for i in range(k))          # row 0 of A times [0, g]
        den = 1 - ef * eb
        fn = [(fi - ef * gi) / den for fi, gi in zip(f + [0], [0] + g)]
        gn = [(gi - eb * fi) / den for fi, gi in zip(f + [0], [0] + g)]
        f, g = fn, gn
        ex = sum(col[k - i] * x[i] for i in range(k))
        x = [xi + (b[k] - ex) * gi for xi, gi in zip(x + [0], g)]
    return np.array([complex(v) for v in x])
