"""Rows, scenes, FP64 reference and FP32 error model of the cross-ambiguity function, shared by
tests/test_caf_envelope_cpu.py and tests/test_caf_envelope_gpu.py.  Imports without a GPU.

Rows: every row of edge_cases.CAF_ROWS (each default (M, M2) kernel instance on both sides of each plan boundary), the
range lengths M = 2^8 ... 2^13 forced through B200DD_CAF_LOG2M, the part splits forced through B200DD_CAF_PARTS,
blah2's config-2 geometry, two off-centre Doppler windows on 1 s CPIs (pre-rotation phase > 10^3 rad) and the config-3
size (2e7 samples).

Scenes (all float32-representable, which is what the device path reads):
  white       random_iq, uniform +-100 I and Q, rounded to float32
  direct      make_scene: int16 reference, direct path + clutter + targets, no clutter filter
  filtered    the same scene through the FP64 clutter filter (oracle), rounded to complex64: what the pipeline hands over
  narrowband  reference = one strong tone on a range-FFT bin (amplitude 3000) + unit noise; surveillance = half of it
              + noise: all energy in one FFT bin and one Doppler bin
  fc32        the direct scene unquantised and scaled by 2^-15, rounded to float32: non-integer full-mantissa samples

Error model
-----------
u = 2^-24.  A rounding to float is off by at most u relative to the value it rounds, and by u / sqrt(3) in rms (a
uniformly distributed rounding error); the roundings of different operations are independent and add in quadrature
(as in tests/test_spectrum_envelope_gpu.py).  So every term below is a variance built from R1 = u^2 / 3 per rounding,
and the bar is LAMBDA sqrt(sum of the variances), LAMBDA = 4: the largest of 10^6 complex Gaussian errors is ~3.7 times
their rms.  ETA^2 = 7 R1 is the variance one radix-2 stage of an FP32 transform adds to one value: three roundings of
the butterfly and a twiddle off by up to two roundings (a table value rounded to float, or on the DIT core the product
of two of them: DESIGN s3).

FFT of length M = 2^l of v, exact output V (unnormalised).  A stage-s error reaches output k through the 2^(l-s)
values of that stage that feed it; by Parseval their energy is P_s(k) = 2^(s-l) sum |V_k'|^2 over the outputs k' they
feed (k' = k mod 2^s), so P_s(k) <= min(2^(s-l) ||V||^2, max|V|^2) and, for the part that comes from V_k itself,
sum_s 2^(s-l) |V_k|^2 < 2 |V_k|^2.  With the stages in quadrature:
    E |dV_k|^2 <= ETA^2 CONE(l, ||V||^2, max|V|^2),  CONE = sum_{s=1..l} min(2^(s-l) ||V||^2, max|V|^2)
    E ||dV (.) G||^2 <= ETA^2 (l ||V||^2 ||G||^2 / M + 2 ||V (.) G||^2)  for an exact weight vector G
(the first term spreads every stage's error evenly over the outputs, the second is the part that stays on the
output's own class, which is what a strong component of G meets: a tone, the direct path).

Range stage, batch i, part p (segments S_p of hop L, range length M), all quantities FP64 (x pre-rotated):
  X_s, Y_s    M-point spectra of the zero-padded x segment and y window;  a_s = Y_s conj(X_s);  Z_p = sum_s a_s;
  r_p = IFFT(Z_p), the part's lags.
  forward transforms        ETA^2 2 sum_s (l ||X_s||^2 ||Y_s||^2 / M + 2 ||a_s||^2) / M^2      (x and y, each segment)
  accumulation              2 R1 (|S_p| + 3) / 2 (||Z_p||^2 + sum_s ||a_s||^2) / M^2
                            (two FMA roundings per component and step on the running sum; partial sums grow linearly
                            for coherent cross-spectra, as a random walk for incoherent ones: sum_t ||Z_t||^2 <=
                            (|S_p| + 1) / 2 (||Z_p||^2 + sum_s ||a_s||^2); one more step for the product itself)
  inverse transform, 1/M    ETA^2 CONE(l, ||Z_p||^2 / M, max|r_p|^2)   (in lag units; 1/M is a power of two: exact)
  sum of the parts          R1 (nParts - 1) (sum_p max |r_p|)^2
  input rounding            R1 ||x_i||_4^2 ||y_i||_4^2 when dopplerMiddle != 0 (x pre-rotated in double, then rounded)
The range bar of row i is LAMBDA sqrt(V_i) + G max_j |R[i, j]| (see below): one number per batch row.

Doppler stage, column j (v = R[:, j] exact, n = nDopplerBins, M2 = 2^l2, chirp c_k = exp(-i pi k^2 / n), b the
wrapped conj chirp, B = FFT_M2(b), W = FFT_M2(v c), Q = W (.) B, q = IFFT_M2(Q) unnormalised, D = the map column):
  range errors              sum_i V_i: the rows' errors are independent, carried through the exact DFT
  chirp pre-multiply        3 R1 ||v||^2      (chirp rounded to float, two roundings of the complex product)
  Bluestein forward         ETA^2 (l2 ||W||^2 ||B||^2 / M2 + 2 ||Q||^2) / M2^2
  d_bhat                    ||W||^2 (ETA^2 CONE(l2, ||B||^2, max|B|^2) + R1 (2n - 1)) / M2^2   (FP32 FFT of the float chirp)
  filter product            2 R1 ||Q||^2 / M2^2
  Bluestein inverse         ETA^2 CONE(l2, ||Q||^2 / M2, max|q / M2|^2)
  chirp post-multiply       3 R1 max|D|^2
(the scales 1/M, 1/M2 are powers of two and the stores take the float result as it is: neither rounds)
Fixed gain error.  The twiddle tables and the chirp are the same for every batch, so their rounding is a fixed
perturbation of the transforms, not an independent one: each spectrum bin has a fixed gain error of rms at most
G = 2 sqrt(4 R1) sqrt(l) (a twiddle off by up to two roundings per stage, in x and in y), which leaks each lag into its
neighbours the same way in every batch.  Where every batch has the same correlation (a direct path, a tone) that
leakage adds up coherently over the batches into the Doppler row that holds them, so it is added linearly, to the
range row of batch i as G max_j |R[i, j]| and to the map row k as G max_j |D[k, j]| (the exact values).
The map bar of cell (k, j) is LAMBDA sqrt(sum of these variances) + G max_j |D[k, j]|: one number per delay column plus
one per Doppler row.  No term depends on the computed map; none on max|map| alone.
"""
import contextlib
import math
import os

import numpy as np
import scipy.fft as sfft

import edge_cases as E
from blah2_b200.scene import make_scene, random_iq
from oracle import blah2_oracle as O

U = 2.0 ** -24
R1 = U ** 2 / 3                 # variance of one rounding
ETA = math.sqrt(7 * R1)         # rms error one transform stage adds to a value, relative to it
LAMBDA = 4.0

SCENES = ("white", "direct", "filtered", "narrowband", "fc32")
CLUTTER = (-2, 20)          # the clutter filter of the filtered scene: taps -2 .. 17 cover the direct path and clutter


def _row(rid, geom, env=None, scenes=SCENES):
    return dict(id=rid, geom=tuple(geom), env=dict(env or {}), scenes=tuple(scenes))


_PART_GEOM = (-5, 60, -20, 20, 100000, 100000, True)        # test_caf_gpu.test_batch_split_into_parts_gives_the_same_map
_PART_GEOM_4096 = (-5, 60, -5, 5, 100000, 100000, True)
PART_SPLITS = [(9, 1), (9, 2), (9, 3), (9, 100), (10, 2), (10, 3), (11, 100), (12, 2)]

ROWS = (
    [_row("edge-" + E.row_id(r), r["geom"]) for r in E.CAF_ROWS]
    + [_row(f"log2m{l}", (-5, 60, -200, 200, 100000, 100000, True), {"B200DD_CAF_LOG2M": str(l)}) for l in range(8, 14)]
    + [_row(f"parts-log2m{l}-{p}", _PART_GEOM_4096 if l == 12 else _PART_GEOM,
            {"B200DD_CAF_LOG2M": str(l), "B200DD_CAF_PARTS": str(p)}) for l, p in PART_SPLITS]
    + [_row("config2", (0, 299, -128, 128, 2000000, 2000000, True)),
       _row("offcentre-up", (-10, 200, -100, 500, 2000000, 2000000, True)),       # dopplerMiddle +200 Hz: 1257 rad
       _row("offcentre-down", (0, 150, -700, 100, 2000000, 2000000, True)),       # dopplerMiddle -300 Hz: 1885 rad
       _row("config3", (0, 511, -256, 256, 10000000, 20000000, True), scenes=("direct",))]
)
FULL_SIZE = {"config3"}


def row_id(r):
    return r["id"]


def cases():
    """(row, scene) pairs in table order."""
    return [(r, s) for r in ROWS for s in r["scenes"]]


def case_id(c):
    return f"{c[0]['id']}-{c[1]}"


@contextlib.contextmanager
def row_env(row):
    """The row's planner overrides in os.environ for the duration (the planner reads them when a handle is made)."""
    old = {k: os.environ.get(k) for k in ("B200DD_CAF_LOG2M", "B200DD_CAF_PARTS")}
    try:
        for k in old:
            os.environ.pop(k, None)
        os.environ.update(row["env"])
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def plan(row):
    """The handle's plan for the row (b200dd_caf_plan, no device): CafGeometry."""
    from blah2_b200 import capi
    with row_env(row):
        return capi.caf_plan(*row["geom"])[0]


# ---------------------------------------------------------------------------------------------------------- scenes
def _c64(v):
    return np.ascontiguousarray(np.asarray(v).astype(np.complex64))


def make_input(row, scene):
    """(x, y) complex64 of the row's n samples."""
    geom = row["geom"]
    fs, n = geom[4], geom[5]
    seed = 1000 + ROWS.index(row)
    if scene == "white":
        x, y = random_iq(n, seed)
        return _c64(x), _c64(y)
    if scene in ("direct", "filtered"):
        sc = make_scene(n, fs, seed=seed)
        x, y = _c64(sc.x), _c64(sc.y)
        if scene == "filtered":
            ok, yf = O.wienerhopf_process(x.astype(np.complex128), y.astype(np.complex128), *CLUTTER)
            assert ok
            y = _c64(yf)
        return x, y
    if scene == "fc32":
        sc = make_scene(n, fs, seed=seed, quantise=False)
        return _c64(sc.x * 2.0 ** -15), _c64(sc.y * 2.0 ** -15)
    if scene == "narrowband":
        M = int(plan(row).range_fft_len)
        rng = np.random.default_rng(seed)
        k0 = M // 8 + 3
        t = (np.arange(n, dtype=np.int64) * k0) % M
        noise = lambda: (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / math.sqrt(2.0)
        x = 3000.0 * np.exp(2j * np.pi * t / M) + noise()
        y = 0.5 * x + noise()
        return _c64(x), _c64(y)
    raise ValueError(scene)


# ------------------------------------------------------------------------------------------------- FP64 reference
def reference(row, x, y):
    """(R, map) in FP64 from the complex128 widening of the complex64 samples, pre-rotation in FP64."""
    og = O.ambiguity_geometry(*row["geom"])
    xr = O.ambiguity_prerotate(x.astype(np.complex128), og)
    R = O.range_matrix(xr, y.astype(np.complex128), og)
    return R, O.doppler_transform(R, og)


# -------------------------------------------------------------------------------------------------- segment layout
def _layout(g, og):
    """Index and mask arrays [nSeg, M] of the x segments and y windows of a batch, and the part of each segment."""
    M, L, nseg, nparts = int(g.range_fft_len), int(g.range_hop), int(g.range_segments), int(g.range_parts)
    nC, nL, lag0 = og.nCorr, og.nDelayBins, og.delayMin
    spp = -(-nseg // nparts)
    assert -(-nseg // spp) == nparts
    s = np.arange(nseg)[:, None]
    m = np.arange(M)[None, :]
    n0 = s * L
    ln = np.minimum(L, nC - n0)
    xi = n0 + m
    xm = m < ln
    yi = n0 + lag0 + m
    ym = (m < ln + nL - 1) & (yi >= 0) & (yi < nC)
    return dict(M=M, L=L, nseg=nseg, nparts=nparts, spp=spp, part=np.arange(nseg) // spp,
                xi=np.where(xm, xi, 0), xm=xm, yi=np.clip(yi, 0, nC - 1), ym=ym)


def _batches(a, og):
    return a[: og.nDopplerBins * og.nCorr].reshape(og.nDopplerBins, og.nCorr)


def _chunk(lay, og):
    return max(1, int(2 ** 24 // (lay["nseg"] * lay["M"])))


# ------------------------------------------------------------------------------------------------------ error model
def cone(l, norm2, inf2):
    """sum_{s=1..l} min(2^(s-l) norm2, inf2) (see the module docstring); arrays broadcast."""
    return sum(np.minimum(2.0 ** (s - l) * norm2, inf2) for s in range(1, int(l) + 1))


def _range_variance_segments(xb, yb, lay, og):
    """Per-row variance of the range stage for rows whose segments are transformed here (hop > 1)."""
    M, nparts, part = lay["M"], lay["nparts"], lay["part"]
    l = math.log2(M)
    nL = og.nDelayBins
    V = np.zeros(xb.shape[0])
    rmax = np.zeros((xb.shape[0], nparts))
    for b0 in range(0, xb.shape[0], _chunk(lay, og)):
        xs = xb[b0:b0 + _chunk(lay, og)][:, lay["xi"]] * lay["xm"]
        ys = yb[b0:b0 + _chunk(lay, og)][:, lay["yi"]] * lay["ym"]
        X = np.fft.fft(xs, axis=-1)
        Y = np.fft.fft(ys, axis=-1)
        a = Y * np.conj(X)
        A2 = np.sum(np.abs(a) ** 2, axis=-1)                                   # [b, s]
        B2 = M * np.sum(np.abs(xs) ** 2, axis=-1) * np.sum(np.abs(ys) ** 2, axis=-1)
        for p in range(nparts):
            sel = part == p
            Z = a[:, sel].sum(axis=1)
            Z2 = np.sum(np.abs(Z) ** 2, axis=-1)
            r = np.fft.ifft(Z, axis=-1)
            rinf = np.max(np.abs(r), axis=-1)
            rmax[b0:b0 + len(Z), p] = np.max(np.abs(r[:, :nL]), axis=-1)
            nS = int(sel.sum())
            sA2 = A2[:, sel].sum(axis=1)
            V[b0:b0 + len(Z)] += (ETA ** 2 * 2 * (l * B2[:, sel] + 2 * A2[:, sel]).sum(axis=1) / M ** 2
                                  + ETA ** 2 * cone(l, Z2 / M, rinf ** 2)
                                  + 2 * R1 * (nS + 3) / 2 * (Z2 + sA2) / M ** 2)
    return V, rmax


def _range_variance_hop1(xb, yb, lay, og):
    """The same for hop 1 (one x sample per segment, X_s = x_n on every bin): closed forms, one correlation per part."""
    M, nparts, spp = lay["M"], lay["nparts"], lay["spp"]
    l = math.log2(M)
    nC, nL, lag0 = og.nCorr, og.nDelayBins, og.delayMin
    V = np.zeros(xb.shape[0])
    rmax = np.zeros((xb.shape[0], nparts))
    ay2 = np.abs(yb) ** 2
    cy = np.concatenate([np.zeros((yb.shape[0], 1)), np.cumsum(ay2, axis=1)], axis=1)
    for p in range(nparts):
        na, nb = p * spp, min(nC, (p + 1) * spp)
        n = np.arange(na, nb)
        lo = np.clip(n + lag0, 0, nC)
        hi = np.clip(n + lag0 + nL, 0, nC)
        ny2 = cy[:, hi] - cy[:, lo]                                          # ||y window||^2 per segment
        A2 = M * np.abs(xb[:, na:nb]) ** 2 * ny2                             # ||a_s||^2 = ||X_s||^2 ||Y_s||^2 / M = B_s^2
        # z_p[m] = sum_n conj(x_n) y[n + lag0 + m], m < nL (zero outside the batch): one FFT correlation
        w0 = na + lag0
        span = (nb - na) + nL - 1
        idx = w0 + np.arange(span)
        seg = np.where((idx >= 0) & (idx < nC), yb[:, np.clip(idx, 0, nC - 1)], 0)
        N = sfft.next_fast_len(span + (nb - na))
        z = np.fft.ifft(np.fft.fft(seg, N, axis=-1) * np.conj(np.fft.fft(xb[:, na:nb], N, axis=-1)), axis=-1)[:, :nL]
        Z2 = M * np.sum(np.abs(z) ** 2, axis=-1)
        rinf = np.max(np.abs(z), axis=-1)
        rmax[:, p] = rinf
        nS = nb - na
        sA2 = A2.sum(axis=1)
        V += (ETA ** 2 * 2 * (l + 2) * sA2 / M ** 2 + ETA ** 2 * cone(l, Z2 / M, rinf ** 2)
              + 2 * R1 * (nS + 3) / 2 * (Z2 + sA2) / M ** 2)
    return V, rmax


def chirp(n):
    k = np.arange(n, dtype=np.int64)
    return np.exp(-1j * np.pi * ((k * k) % (2 * n)) / n)


def error_model(row, g, x, y, R):
    """(range bar [nDop], map bar [nDop, nDel] in the map's row order) for complex64 inputs x, y; R is the FP64
    range matrix of reference()."""
    og = O.ambiguity_geometry(*row["geom"])
    lay = _layout(g, og)
    xr = O.ambiguity_prerotate(x.astype(np.complex128), og)
    xb, yb = _batches(xr, og), _batches(y.astype(np.complex128), og)
    if lay["L"] == 1:
        V, rmax = _range_variance_hop1(xb, yb, lay, og)
    else:
        V, rmax = _range_variance_segments(xb, yb, lay, og)
    V += R1 * (lay["nparts"] - 1) * np.sum(rmax, axis=1) ** 2
    if og.dopplerMiddle != 0:
        V += R1 * np.sqrt(np.sum(np.abs(xb) ** 4, axis=1)) * np.sqrt(np.sum(np.abs(yb) ** 4, axis=1))
    gain = 2 * math.sqrt(4 * R1) * math.sqrt(math.log2(lay["M"]))
    range_bar = LAMBDA * np.sqrt(V) + gain * np.max(np.abs(R), axis=1)
    # Doppler stage
    n, M2 = og.nDopplerBins, int(g.doppler_fft_len)
    l2 = math.log2(M2)
    c = chirp(n)
    b = np.zeros(M2, dtype=np.complex128)
    b[:n] = np.conj(c)
    b[M2 - np.arange(1, n)] = np.conj(c[1:])
    Bh = np.fft.fft(b)
    B2, Binf = float(np.sum(np.abs(Bh) ** 2)), float(np.max(np.abs(Bh)))
    v2 = np.sum(np.abs(R) ** 2, axis=0)
    W = np.fft.fft(R * c[:, None], M2, axis=0)
    W2 = np.sum(np.abs(W) ** 2, axis=0)
    Q = W * Bh[:, None]
    Q2 = np.sum(np.abs(Q) ** 2, axis=0)
    qinf = np.max(np.abs(np.fft.ifft(Q, axis=0)), axis=0) * M2
    Dinf = np.max(np.abs(np.fft.fft(R, axis=0)), axis=0)
    Vb = ((ETA ** 2 * (l2 * W2 * B2 / M2 + 2 * Q2) + W2 * (ETA ** 2 * cone(l2, B2, Binf ** 2) + R1 * (2 * n - 1))
           + 2 * R1 * Q2) / M2 ** 2 + ETA ** 2 * cone(l2, Q2 / M2, (qinf / M2) ** 2)
          + 3 * R1 * v2 + 3 * R1 * Dinf ** 2)
    D = O.doppler_transform(R, og)
    map_bar = LAMBDA * np.sqrt(np.sum(V) + Vb)[None, :] + gain * np.max(np.abs(D), axis=1)[:, None]
    return range_bar, map_bar


# ----------------------------------------------------------------------------------- numpy FP32 restatement (CPU)
def affordable(row, g):
    """Rows whose FP32 restatement transforms fewer than 3e8 points."""
    og = O.ambiguity_geometry(*row["geom"])
    return og.nDopplerBins * int(g.range_segments) * int(g.range_fft_len) <= 3e8 and row["id"] not in FULL_SIZE


def restate_fp32(row, g, x, y):
    """(R, map) by the kernels' algorithm in FP32: pre-rotation in double rounded to float, complex64 FFTs per
    segment, cross-spectra accumulated in complex64 in segment order per part, one inverse per part, the parts added in
    order, then Bluestein in complex64 with a float chirp and a complex64 filter spectrum."""
    og = O.ambiguity_geometry(*row["geom"])
    lay = _layout(g, og)
    M, nparts, part = lay["M"], lay["nparts"], lay["part"]
    nD, nL = og.nDopplerBins, og.nDelayBins
    xr = _c64(O.ambiguity_prerotate(x.astype(np.complex128), og))
    xb, yb = _batches(xr, og), _batches(y, og)
    R = np.zeros((nD, nL), dtype=np.complex64)
    xm, ym = lay["xm"].astype(np.complex64), lay["ym"].astype(np.complex64)
    for b0 in range(0, nD, _chunk(lay, og)):
        b1 = min(nD, b0 + _chunk(lay, og))
        X = sfft.fft(xb[b0:b1][:, lay["xi"]] * xm, axis=-1)
        Y = sfft.fft(yb[b0:b1][:, lay["yi"]] * ym, axis=-1)
        assert X.dtype == np.complex64
        acc = None
        for p in range(nparts):
            Z = np.zeros((b1 - b0, M), dtype=np.complex64)
            for s in np.nonzero(part == p)[0]:
                Z = Z + Y[:, s] * np.conj(X[:, s])
            r = sfft.ifft(Z, axis=-1)[:, :nL]
            acc = r if acc is None else acc + r
        R[b0:b1] = acc
    M2 = int(g.doppler_fft_len)
    c = _c64(chirp(nD))
    b = np.zeros(M2, dtype=np.complex64)
    b[:nD] = np.conj(c)
    b[M2 - np.arange(1, nD)] = np.conj(c[1:])
    Bh = sfft.fft(b)
    q = sfft.ifft(sfft.fft(R * c[:, None], M2, axis=0) * Bh[:, None], axis=0)[:nD] * c[:, None]
    assert q.dtype == np.complex64
    return R, q[(np.arange(nD) + nD // 2 + 1) % nD]


# ----------------------------------------------------------------------------------------------------- map products
def db_bar(ref, bar):
    """|10 log10|z| - 10 log10|ref|| bound for |z - ref| <= bar, cell by cell."""
    a = np.abs(ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(a > bar, -10.0 * np.log10(1.0 - bar / a), np.inf)


def cfar_margins(m, delay, doppler, pfa, nGuard, nTrain, minDelay, minDoppler):
    """(decision, sq - thr, training-cell count) of every cell, as edge_cases.cfar_1d decides them."""
    m = np.asarray(m, dtype=np.complex128)
    sq = np.abs(m * m)
    nDop, nDel = m.shape
    j = np.arange(nDel)
    noise = np.zeros(m.shape)
    cells = np.zeros(nDel, dtype=np.int64)
    offs = [(d, True) for d in range(-nGuard - nTrain, -nGuard)] + [(d, False) for d in range(nGuard + 1, nGuard + nTrain + 1)]
    for d, leading in offs:
        k = j + d
        ok = (k > 0 if leading else k >= 0) & (k < nDel)
        sh = np.zeros(m.shape)
        sh[:, ok] = sq[:, k[ok]]
        noise = noise + sh
        cells += ok
    alpha = np.array([k * (math.pow(pfa, -1.0 / k) - 1) if k else np.nan for k in range(int(cells.max(initial=0)) + 1)])
    with np.errstate(invalid="ignore"):
        thr = alpha[cells] * (noise / np.where(cells > 0, cells, 1))
    det = (sq > thr) & (cells > 0)
    det &= (np.asarray(delay) >= minDelay)[None, :]
    det &= ~(np.abs(np.asarray(doppler)) < minDoppler)[:, None]
    return det, sq - thr, cells, alpha


def cfar_slack(ref, bar, nGuard, nTrain, alpha, cells):
    """Bound on |d(sq - thr)| when every cell moves by at most its bar: |z|^2 moves by <= 2|z| b + b^2, the
    threshold by alpha times the mean of that over the training cells."""
    a = np.abs(ref)
    dsq = 2 * a * bar + bar ** 2
    nDel = ref.shape[1]
    j = np.arange(nDel)
    tot = np.zeros(ref.shape)
    offs = [(d, True) for d in range(-nGuard - nTrain, -nGuard)] + [(d, False) for d in range(nGuard + 1, nGuard + nTrain + 1)]
    for d, leading in offs:
        k = j + d
        ok = (k > 0 if leading else k >= 0) & (k < nDel)
        sh = np.zeros(ref.shape)
        sh[:, ok] = dsq[:, k[ok]]
        tot += sh
    with np.errstate(invalid="ignore"):
        return dsq + np.nan_to_num(alpha[cells]) * tot / np.where(cells > 0, cells, 1)
