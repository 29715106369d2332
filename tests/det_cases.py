"""Detection-tail cases whose decisions sit exactly on a boundary, and a restatement of CFAR, Centroid and Interpolate
that takes each cell's values as given.

The restatement follows the reference's order of operations (CfarDetector1D.cpp:23-100, Centroid.cpp:19-73,
Interpolate.cpp:20-91) in Python floats, so every operation is one IEEE double rounding.  It reads two per-cell
arrays instead of the map:

  sq[r][c]  |z z| = hypot(re^2 - im^2, 2 re im), the CFAR statistic;
  db[r][c]  10 log10|z| - noisePower, the value CFAR emits as SNR and Interpolate fits its parabola to.

Fed with values computed by the CPU's libm it is the reference; fed with the device's own per-cell values (the map
document's cell_db, CUDA's hypot) it is what the kernels must compute bit for bit, with no libm difference left.

``fault`` plants one wrong change in a stage, so a test can show that a case set tells the right code from it:

  cfar_ge            CFAR detects at sq == threshold (>= for >)
  train_right_first  CFAR sums the right training window before the left one
  alpha_shift        CFAR reads alpha[nCells - 1]
  alpha_f32          CFAR's alpha table held in float
  centroid_le        Centroid drops a detection at equal SNR (<= for <)
  centroid_dmin_ge   Centroid counts a neighbour at exactly delay - nDelay (>= for >)
  centroid_fma       Centroid's Doppler window edges as one fused multiply-add each
  interp_le          Interpolate drops a plateau (s1 <= s0 for s1 < s0)
  interp_den         Interpolate's denominator reassociated: 2 ((s0 + s2) - 2 s1)
  snr_fma            every dB value as fma(log10|z|, 10, -noisePower) (the contracted form det.cu once compiled to)

Interpolate drops a detection whose neighbour cells fall outside the map, as det.cu does; the reference reads out of
bounds there (undefined behaviour), so cases that reach the fence are marked ``fenced`` and only compared with the
device.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

PFA = 2.0 ** -16
# alpha[n] = n (pfa^(-1/n) - 1) is exact for pfa = 2^-16 when -1/n is: pfa^(-1/n) = 2^(16/n)
ALPHA_EXACT = {1: 65535.0, 2: 510.0, 4: 60.0, 8: 24.0, 16: 16.0}
NOISE = 14.73  # a noisePower that is not 0, so a fused and a twice-rounded dB value differ

CFAR_FAULTS = ("cfar_ge", "train_right_first", "alpha_shift", "alpha_f32")
CENTROID_FAULTS = ("centroid_le", "centroid_dmin_ge", "centroid_fma")
INTERP_FAULTS = ("interp_le", "interp_den")


def int8(v: int) -> int:
    v = int(v) & 0xFF
    return v - 256 if v >= 128 else v


def rn(q: Fraction) -> float:
    """q rounded to the nearest double (ties to even)."""
    return float(q)


def fma(a: float, b: float, c: float) -> float:
    return rn(Fraction(a) * Fraction(b) + Fraction(c))


def alpha(n: int, pfa: float) -> float:
    return n * (math.pow(pfa, -1.0 / n) - 1)  # CfarDetector1D.cpp:76


# ---------------------------------------------------------------------------------------------- per-cell values
def sq_values(m: np.ndarray, hypot=np.hypot) -> np.ndarray:
    """|z z| of every cell: the complex square in separately rounded operations, then hypot (the CPU's by default)."""
    re = m.real * m.real - m.imag * m.imag
    im = m.real * m.imag + m.imag * m.real
    return np.asarray(hypot(re, im), dtype=np.float64)


def log10_abs(m: np.ndarray) -> np.ndarray:
    """log10|z| of every cell with the CPU's libm (math.log10 is the C library's log10; numpy's may differ)."""
    a = np.abs(m).ravel()
    out = np.array([math.log10(v) if v > 0 else (-math.inf if v == 0 else math.nan) for v in a.tolist()])
    return out.reshape(m.shape)


def db_values(L: np.ndarray, noise: float, fused: bool = False) -> np.ndarray:
    """10 log10|z| - noise from log10|z|: both operations rounded, or (fused) one fma."""
    if not fused:
        return (10.0 * L) - noise
    out = np.empty(L.shape)
    for idx, v in np.ndenumerate(L):
        out[idx] = fma(float(v), 10.0, -noise) if math.isfinite(v) else 10.0 * v - noise
    return out


# ---------------------------------------------------------------------------------------------- restatement
def train_cells(j: int, nDel: int, nGuard: int, nTrain: int):
    left = [k for k in range(j - nGuard - nTrain, j - nGuard) if 0 < k < nDel]       # :59-64 (k > 0)
    right = [k for k in range(j + nGuard + 1, j + nGuard + nTrain + 1) if 0 <= k < nDel]  # :66-71
    return left, right


def threshold(sqrow, j, nGuard, nTrain, pfa, fault=None):
    """alpha * (sequential training sum / nCells) of column j, or None where nCells == 0 (alpha is NaN)."""
    left, right = train_cells(j, len(sqrow), nGuard, nTrain)
    idx = right + left if fault == "train_right_first" else left + right
    n = len(idx)
    if n == 0:
        return None
    if fault == "alpha_shift":
        a = alpha(n - 1, pfa) if n > 1 else 0.0  # the device table's alpha[0] is 0
    else:
        a = alpha(n, pfa)
    if fault == "alpha_f32":
        a = float(np.float32(a))
    s = 0.0
    for k in idx:
        s += float(sqrow[k])
    s /= n
    return a * s


def cfar(sq, db, delay, doppler, pfa, nGuard, nTrain, minDelay, minDoppler, fault=None):
    nGuard, nTrain, minDelay = int8(nGuard), int8(nTrain), int8(minDelay)
    nDop, nDel = sq.shape
    od, of, os_ = [], [], []
    for i in range(nDop):
        if abs(float(doppler[i])) < minDoppler:  # :40
            continue
        row = [float(v) for v in sq[i]]
        for j in range(nDel):
            if int(delay[j]) < minDelay:  # :53
                continue
            t = threshold(row, j, nGuard, nTrain, pfa, fault)
            if t is None:
                continue
            hit = row[j] >= t if fault == "cfar_ge" else row[j] > t  # :86
            if hit:
                od.append(float(j + int(delay[0])))
                of.append(float(doppler[i]))
                os_.append(float(db[i][j]))
    return np.asarray(od, dtype=np.float64), np.asarray(of, dtype=np.float64), np.asarray(os_, dtype=np.float64)


def centroid(delay, doppler, snr, nDelay, nDoppler, res, fault=None):
    nDelay &= 0xFFFF
    nDoppler &= 0xFFFF
    d = np.asarray(delay, dtype=np.float64)
    f = np.asarray(doppler, dtype=np.float64)
    s = np.asarray(snr, dtype=np.float64)
    keep = np.ones(d.size, dtype=bool)
    span = nDoppler * res
    for i in range(d.size):
        dmin = (int(d[i]) - nDelay) & 0xFFFF  # uint16_t (Centroid.cpp:28,34-35)
        dmax = (int(d[i]) + nDelay) & 0xFFFF
        if fault == "centroid_fma":
            fmin, fmax = fma(-float(nDoppler), res, float(f[i])), fma(float(nDoppler), res, float(f[i]))
        else:
            fmin, fmax = float(f[i]) - span, float(f[i]) + span
        lo = d >= dmin if fault == "centroid_dmin_ge" else d > dmin
        near = lo & (d < dmax) & (f > fmin) & (f < fmax)
        near[i] = False
        higher = s[i] <= s if fault == "centroid_le" else s[i] < s
        keep[i] = not np.any(near & higher)
    return d[keep], f[keep], s[keep]


def hz_to_bin(axis, hz) -> int:
    """Map::doppler_hz_to_bin (Map.cpp:103-113): the first exact match, 0 when there is none."""
    for k, v in enumerate(axis):
        if v == hz:
            return k
    return 0


def _parabola(s0, s1, s2, fault):
    num = s0 - s2
    den = 2 * ((s0 + s2) - (2 * s1)) if fault == "interp_den" else 2 * ((s0 - (2 * s1)) + s2)
    off = num / den if den != 0 else (math.nan if num == 0 or math.isnan(num) else math.copysign(math.inf, num) * math.copysign(1.0, den))
    return off, s1 - ((num * off) / 4)


def _lt(a, b, fault):
    return a <= b if fault == "interp_le" else a < b


def interpolate(delay, doppler, snr, db, mdelay, mdoppler, doDelay=True, doDoppler=True, fault=None):
    """Interpolate::process on the cell values db, with det.cu's fence (see the module doc).  Returns the three lists
    and, per input detection, whether the fence dropped it."""
    nDop, nDel = db.shape
    d0, dl = float(mdelay[0]), float(mdelay[-1])
    od, of, os_, fenced = [], [], [], []
    for i in range(len(snr)):
        d, f, s = float(delay[i]), float(doppler[i]), float(snr[i])
        intDelay, intDoppler, intSnrDelay, intSnrDoppler = d, f, s, s
        row = hz_to_bin(mdoppler, f)
        c = int(d - d0)
        fence = False
        if doDelay:
            if d == d0 or d == dl:  # :46-49
                fenced.append(False)
                continue
            if c - 1 < 0 or c + 1 >= nDel:
                fenced.append(True)
                continue
            s0, s1, s2 = float(db[row][c - 1]), float(db[row][c]), float(db[row][c + 1])  # :50-52
            if _lt(s1, s0, fault) or _lt(s1, s2, fault):  # :54-58
                fenced.append(False)
                continue
            off, intSnrDelay = _parabola(s0, s1, s2, fault)
            intDelay = d + off
        if doDoppler:
            if f == float(mdoppler[0]) or f == float(mdoppler[-1]):  # :67-70
                fenced.append(False)
                continue
            if row - 1 < 0 or row + 1 >= nDop or c < 0 or c >= nDel:
                fenced.append(True)
                continue
            s0, s1, s2 = float(db[row - 1][c]), float(db[row][c]), float(db[row + 1][c])  # :71-73
            if _lt(s1, s0, fault) or _lt(s1, s2, fault):  # :75-78
                fenced.append(False)
                continue
            off, intSnrDelay = _parabola(s0, s1, s2, fault)  # :80 (sic: intSnrDelay)
            intDoppler = f + ((float(mdoppler[1]) - float(mdoppler[0])) * off)
        fenced.append(fence)
        od.append(intDelay)
        of.append(intDoppler)
        os_.append(max(max(intSnrDelay, intSnrDoppler), s))  # :86, std::max keeps a NaN first argument
    return (np.asarray(od, dtype=np.float64), np.asarray(of, dtype=np.float64), np.asarray(os_, dtype=np.float64),
            np.asarray(fenced, dtype=bool))


def chain(sq, db, delay, doppler, p, last=3, fault=None):
    """CFAR -> Centroid -> Interpolate of blah2.cpp:285-287 with the handle parameters p (see det_params)."""
    d1 = cfar(sq, db, delay, doppler, p["pfa"], p["nGuard"], p["nTrain"], p["minDelay"], p["minDoppler"], fault)
    if last == 1:
        return d1
    d2 = centroid(*d1, p["nCentroidDelay"], p["nCentroidDoppler"], p["resolutionDoppler"], fault)
    if last == 2:
        return d2
    return interpolate(*d2, db, delay, doppler, p.get("doDelay", True), p.get("doDoppler", True), fault)[:3]


def same(a, b) -> bool:
    """Two detection lists equal bit for bit (NaN where NaN)."""
    return len(a[0]) == len(b[0]) and all(
        np.array_equal(np.asarray(x, np.float64), np.asarray(y, np.float64), equal_nan=True) for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------- CFAR cases
def _f32_next(x, toward):
    return float(np.nextafter(np.float32(x), np.float32(toward)))


def hug(T, f32=False):
    """Cell magnitudes x > 0 around the threshold T: (at, below, above) with x*x == T (None when no such x exists),
    the largest x*x < T and the smallest x*x > T, for x a double or (f32) a float32."""
    if f32:
        x0 = np.float32(math.sqrt(T))
        cand = [float(x0)]
        for d in (np.float32(0), np.float32(np.inf)):
            x = x0
            for _ in range(3):
                x = np.nextafter(x, d)
                cand.append(float(x))
    else:
        x0 = math.sqrt(T)
        cand = [x0]
        for d in (0.0, math.inf):
            x = x0
            for _ in range(6):
                x = math.nextafter(x, d)
                cand.append(x)
    at = next((x for x in cand if x * x == T), None)
    below = max((x for x in cand if x * x < T), key=lambda x: x * x)
    above = min((x for x in cand if x * x > T), key=lambda x: x * x)
    return at, below, above


def _axis_doppler(n, minDoppler):
    """A strictly increasing Doppler axis of n >= 4 rows whose first rows are -minDoppler, the two doubles either
    side of it, and +minDoppler."""
    below = math.nextafter(minDoppler, 0.0)
    head = [-minDoppler, -below, below, minDoppler]
    return np.asarray(head + [minDoppler + 10.0 * k for k in range(1, n - 3)], dtype=np.float64)[:n]


def det_params(pfa=PFA, nGuard=2, nTrain=8, minDelay=-128, minDoppler=0.0, nCentroidDelay=2, nCentroidDoppler=2,
               resolutionDoppler=10.0, doDelay=True, doDoppler=True):
    return dict(pfa=pfa, nGuard=nGuard, nTrain=nTrain, minDelay=minDelay, minDoppler=minDoppler,
                nCentroidDelay=nCentroidDelay, nCentroidDoppler=nCentroidDoppler, resolutionDoppler=resolutionDoppler,
                doDelay=doDelay, doDoppler=doDoppler)


def cfar_cases():
    """Maps of real-valued cells (the complex square is x^2 and |z| is |x|) with cells under test at, just below and
    just above their thresholds.  Each case: name, map (complex128), delay, doppler, params (as given to the handle,
    before the reference's int8 narrowing), f32 (every cell a float32), ties [(row, col, kind, T)]."""
    cases = []
    rng = np.random.default_rng(2024)

    # 1. float32 maps: ties where nCells is 16 and 8 (alpha 16 and 24); rows at |doppler| == minDoppler and one
    #    ulp inside it; columns at delay == minDelay and one below; the int8 narrowing of nGuard = 258, nTrain = 264,
    #    minDelay = 261 (2, 8 and 5)
    nDel, nGuard, nTrain, minDelay, minDoppler, delay0 = 48, 2, 8, 5, 15.0, -3
    plans = [  # (squares of the background cells, column under test)
        (np.ones(nDel), 24),                                           # nCells 16: T = 16, x = 4
        (np.full(nDel, 4.0), 30),                                      # nCells 16: T = 64, x = 8
        (np.array([1, 4, 9, 16, 4, 4, 9, 1] * 6, float), nDel - 1),    # nCells 8 (left window only): T = 144, x = 12
    ]
    rows, ties = [], []
    for k in range(4):  # rows -15, -(15 - ulp), 15 - ulp, 15: a cell far above its threshold in each
        r = np.ones(nDel)
        r[20 + k] = 100.0
        rows.append(r)
    for bg, j in plans:
        T = threshold(list(bg), j, nGuard, nTrain, PFA)
        for kind, x in zip(("at", "below", "above"), hug(T, f32=True)):
            r = np.sqrt(bg)
            r[j] = x
            ties.append((len(rows), j, kind, T))
            rows.append(r)
    jm = minDelay - delay0  # delay[jm] == minDelay is tested, delay[jm - 1] is skipped (both far above threshold)
    for j in (jm, jm - 1):
        r = np.ones(nDel)
        r[j] = 64.0
        rows.append(r)
    m = np.asarray(rows, dtype=np.float64)
    cases.append(dict(name="f32_ties", map=m.astype(np.complex128), delay=np.arange(delay0, delay0 + nDel, dtype=np.int32),
                      doppler=_axis_doppler(len(rows), minDoppler),
                      params=det_params(nGuard=nGuard + 256, nTrain=nTrain + 256, minDelay=minDelay + 256,
                                        minDoppler=minDoppler), f32=True, ties=ties))

    # 2. window edges: for every map width 1 .. 2 nTrain + 2 nGuard + 2, every column under test at, below and above
    #    its threshold over mixed float32 training cells (nCells runs through 0 .. 16, column 1 shows k > 0)
    nGuard, nTrain = 1, 8
    for nDel in range(1, 2 * nTrain + 2 * nGuard + 3):
        rows, ties = [], []
        for j in range(nDel):
            bg = rng.choice([0.5, 1.0, 1.25, 2.0, 3.0], size=nDel)
            T = threshold(list(bg * bg), j, nGuard, nTrain, PFA)
            if T is None:
                rows.append(bg.copy())
                continue
            for kind, x in zip(("at", "below", "above"), hug(T)):
                if x is None:
                    continue
                r = bg.copy()
                r[j] = x
                ties.append((len(rows), j, kind, T))
                rows.append(r)
        m = np.asarray(rows, dtype=np.float64)
        cases.append(dict(name=f"edges_w{nDel}", map=m.astype(np.complex128), delay=np.arange(nDel, dtype=np.int32),
                          doppler=np.arange(len(rows), dtype=np.float64) * 10.0 - 5.0,
                          params=det_params(nGuard=nGuard, nTrain=nTrain), f32=False, ties=ties))

    # 3. mixed magnitudes: a 2^54 training cell whose small companions the sequential sum loses, so left-then-right,
    #    right-then-left, pairwise and exact sums differ; the cell under test between the thresholds
    nDel, nGuard, nTrain, j = 40, 2, 8, 20
    small = 1.375  # square 1.890625 < ulp(2^54) / 2
    rows, ties = [], []
    for big_at in ("left_first", "right_first", "right_last", "left_last"):
        bg = np.full(nDel, small)
        left, right = train_cells(j, nDel, nGuard, nTrain)
        k = {"left_first": left[0], "right_first": right[0], "right_last": right[-1], "left_last": left[-1]}[big_at]
        bg[k] = 2.0 ** 27
        sqrow = list(bg * bg)
        T = threshold(sqrow, j, nGuard, nTrain, PFA)
        Tr = threshold(sqrow, j, nGuard, nTrain, PFA, "train_right_first")
        for kind, x in zip(("at", "below", "above"), hug(T)):
            if x is None:
                continue
            r = bg.copy()
            r[j] = x
            ties.append((len(rows), j, kind, T))
            rows.append(r)
        # strictly between the two sequential orders
        lo, hi = min(T, Tr), max(T, Tr)
        x = math.sqrt(lo)
        while x * x <= lo:
            x = math.nextafter(x, math.inf)
        if x * x < hi:
            r = bg.copy()
            r[j] = x
            ties.append((len(rows), j, "between", T))
            rows.append(r)
    m = np.asarray(rows, dtype=np.float64)
    cases.append(dict(name="mixed_windows", map=m.astype(np.complex128), delay=np.arange(nDel, dtype=np.int32),
                      doppler=np.arange(len(rows), dtype=np.float64) - 2.0, params=det_params(nGuard=nGuard, nTrain=nTrain),
                      f32=False, ties=ties))
    return cases


# ---------------------------------------------------------------------------------------------- Centroid cases
CENTROID_PARAMS = dict(nDelay=4, nDoppler=3, res=0.1)  # nDoppler * res = 0.30000000000000004: inexact


def _fma_window_miss():
    """A Doppler value f where the fused window edge fma(-3, 0.1, f) differs from rn(f - rn(3 * 0.1))."""
    span = 3 * 0.1
    for k in range(1, 10000):
        f = 0.2 + k * 0.0137
        if fma(-3.0, 0.1, f) != f - span:
            return f
    raise AssertionError("no Doppler value separates the fused window edge")


def centroid_cases():
    """Detection lists (name, delay, doppler, snr) for Centroid(4, 3, 0.1)."""
    nD = CENTROID_PARAMS["nDelay"]
    span = 3 * 0.1
    cases = []
    f0 = 50.0
    # a neighbour of higher SNR at exactly delay -/+ nDelay (outside), at delay -/+ (nDelay - 1) (inside)
    for dd in (-nD, nD, -(nD - 1), nD - 1):
        cases.append((f"delay_edge_{dd:+d}", [100.0, 100.0 + dd], [f0, f0], [10.0, 11.0]))
    # a neighbour at exactly rn(f -/+ nDoppler res) (outside) and one ulp inside it
    for sgn in (-1, 1):
        edge = f0 - span if sgn < 0 else f0 + span
        inside = math.nextafter(edge, f0)
        cases.append((f"doppler_edge_{sgn:+d}", [100.0, 100.0], [f0, edge], [10.0, 11.0]))
        cases.append((f"doppler_inside_{sgn:+d}", [100.0, 100.0], [f0, inside], [10.0, 11.0]))
    # where the fused edge differs: a neighbour exactly at the twice-rounded edge and at the fused one
    f1 = _fma_window_miss()
    for edge in (f1 - span, fma(-3.0, 0.1, f1), f1 + span, fma(3.0, 0.1, f1)):
        cases.append((f"doppler_fma_{edge!r}", [100.0, 100.0], [f1, edge], [10.0, 11.0]))
    # equal SNRs: both kept
    cases.append(("equal_snr", [100.0, 101.0, 102.0], [f0, f0, f0 + 0.1], [7.5, 7.5, 7.5]))
    # uint16 edges: below 0 (delayMin wraps high, nothing lies above it), at and above 65536 (delayMax wraps low),
    # negative delays
    cases.append(("wrap_low", [2.0, 3.0, 1.0, 0.0], [f0] * 4, [5.0, 9.0, 7.0, 8.0]))
    cases.append(("wrap_high", [65533.0, 65534.0, 65535.0, 65536.0, 65537.0], [f0] * 5, [5.0, 9.0, 7.0, 8.0, 6.0]))
    cases.append(("negative", [-3.0, -2.0, -1.0, -7.0, -6.5], [f0] * 5, [5.0, 9.0, 7.0, 8.0, 6.0]))
    # list lengths across the 1024-thread compaction: clusters of near detections with some equal SNRs
    rng = np.random.default_rng(77)
    for n in (1, 1023, 1024, 1025, 2049):
        d = rng.integers(0, 400, n).astype(np.float64)
        f = np.round(rng.uniform(-20, 20, n), 1)
        s = np.round(rng.uniform(0, 20, n), 0)
        cases.append((f"random_{n}", d, f, s))
    return [(name, np.asarray(d, np.float64), np.asarray(f, np.float64), np.asarray(s, np.float64))
            for name, d, f, s in cases]


# ---------------------------------------------------------------------------------------------- Interpolate cases
def plateau_pairs(count=16, noise=NOISE, seed=5):
    """count different plateau pairs (see plateau_pair): a libm whose log10 differs in the last place keeps some."""
    return [plateau_pair(noise, seed + k) for k in range(count)]


def plateau_pair(noise=NOISE, seed=5):
    """Magnitudes a > b > 0 with log10 b < log10 a but rn(10 log10 a) == rn(10 log10 b) (CPU libm), where the
    fused dB values differ: fma(log10 b, 10, -noise) < fma(log10 a, 10, -noise).  A cell b between a and a smaller
    cell is then a plateau peak for the reference and a drop for the fused form."""
    rng = np.random.default_rng(seed)
    for _ in range(100000):
        a = float(rng.uniform(1e3, 1e5))
        b = a
        for _ in range(64):
            b = math.nextafter(b, 0.0)
            La, Lb = math.log10(a), math.log10(b)
            if Lb < La and 10.0 * La == 10.0 * Lb and fma(Lb, 10.0, -noise) < fma(La, 10.0, -noise):
                return a, b
            if 10.0 * Lb != 10.0 * La:
                break
    raise AssertionError("no plateau pair found")


def interp_case(noise=NOISE, pair=None):
    """One map of real-valued cells, 5 Doppler rows by 40 delay columns, and a detection list over it: patterns around
    each detection's cell in row 2 (delay neighbours) and column (Doppler neighbours).  Returns a dict with map,
    delay, doppler, list (delay, doppler, snr) and noise."""
    nDop, nDel = 5, 40
    a, b = pair if pair is not None else plateau_pair(noise)
    rng = np.random.default_rng(11)
    m = rng.uniform(1.0, 2.0, (nDop, nDel))
    delay = np.arange(-4, -4 + nDel, dtype=np.int32)
    doppler = np.array([-20.0, -10.0, 0.0, 10.0, 20.0])
    patterns = [  # (left, centre, right) along delay in row 2; (up, down) along Doppler in the centre's column
        ((30.0, 30.0, 10.0), (5.0, 6.0)),     # s1 == s0
        ((10.0, 30.0, 30.0), (6.0, 5.0)),     # s1 == s2
        ((10.0, 30.0, 10.0), (30.0, 7.0)),    # s0 == s2 along delay (offset 0); s1 == s0 along Doppler
        ((30.0, 30.0, 30.0), (30.0, 30.0)),   # all equal: 0 / 0
        ((a, b, 10.0), (b, 10.0)),            # plateau pair along delay and along Doppler
        ((10.0, b, a), (10.0, a)),            # plateau pair, mirrored
        ((11.0, 37.0, 23.0), (19.0, 29.0)),   # generic peak
        ((13.0, 41.0, 17.0), (41.0 * 0.999, 12.0)),
        ((12.0, 25.0, 26.0), (3.0, 4.0)),     # not a peak along delay
        ((3.0, 31.0, 4.0), (33.0, 4.0)),      # not a peak along Doppler
    ]
    cols = []
    for k, ((l, c, r), (u, dn)) in enumerate(patterns):
        j = 2 + 3 * k
        m[2, j - 1:j + 2] = (l, c, r)
        m[1, j], m[3, j] = u, dn
        cols.append(j)
    det = [(float(delay[j]), 0.0) for j in cols]
    # axis ends: first and last delay, first and last Doppler row; a Doppler value off the axis (row 0)
    det += [(float(delay[0]), 0.0), (float(delay[-1]), 0.0), (float(delay[35]), -20.0), (float(delay[35]), 20.0),
            (float(delay[36]), 5.0), (float(delay[37]), -10.0)]
    L = log10_abs(m.astype(np.complex128))
    dbv = db_values(L, noise)
    snr = [float(dbv[hz_to_bin(doppler, f)][int(d - delay[0])]) for d, f in det]
    return dict(map=m.astype(np.complex128), delay=delay, doppler=doppler, noise=noise,
                list=(np.array([d for d, _ in det]), np.array([f for _, f in det]), np.array(snr)), pair=(a, b))


def spike_map(n_det, nDel=256, every=8):
    """A float32 map with exactly n_det isolated spikes CFAR(2^-16, nGuard 1, nTrain 2) detects, in rows of nDel // every,
    their heights varied so Centroid(2, 2, 10) drops some and keeps equal ones."""
    per = nDel // every
    nDop = (n_det + per - 1) // per
    m = np.ones((nDop, nDel))
    k = 0
    for i in range(nDop):
        for j in range(every // 2, nDel, every):
            if k == n_det:
                break
            m[i, j] = 100.0 + (i % 3) + ((j // every) % 2) * 0.5
            m[i, j + 1] = 5.0 + (i % 2)  # an asymmetric shoulder below its own threshold, so Interpolate moves the peak
            k += 1
    return m.astype(np.complex128), np.arange(nDel, dtype=np.int32), np.arange(nDop, dtype=np.float64) * 10.0 - 100.0
