"""Case tables and fast restatements shared by tests/test_kernel_edges_cpu.py and tests/test_kernel_edges_gpu.py.

The default planners pick a kernel instance from the geometry: the range FFT length M from (nDelayBins, nCorr)
(plan_range, caf.cu) and the Bluestein length M2 = the smallest power of two >= 2 nDopplerBins - 1.  The rows below
sit on both sides of every boundary between instances; test_kernel_edges_cpu.py proves with b200dd_caf_plan that
together they reach every default (M, M2) instance, and test_kernel_edges_gpu.py checks each against the oracle.

The detection restatements (cfar_1d, centroid) are vectorised over the whole map / list, so that maps of 10^6 - 10^7
cells can be checked; they are pinned against oracle/blah2_oracle.py on the CPU.
"""
import math

import numpy as np

from oracle import blah2_oracle as O


# ---------------------------------------------------------------------------------------------------- CAF geometries
def _doppler_row(D, n_corr, m2):
    n = (2 * D + 1) * n_corr   # fs = n: 1 Hz resolution, nDopplerBins = 2 D + 1, nCorr = n_corr
    return dict(geom=(-3, 17, -D, D, n, n, True), n_dop=2 * D + 1, n_corr=n_corr, n_del=21, M=256, M2=m2)


def _delay_row(n_del, M):
    n_corr = n_del + 100       # every lag stays inside the oracle's nfft (range_matrix reads z[:, nfft + lag])
    n = 31 * n_corr            # dopplerMax 15 at fs = n: 31 bins
    return dict(geom=(-10, n_del - 11, -15, 15, n, n, True), n_dop=31, n_corr=n_corr, n_del=n_del, M=M, M2=256)


# the planner moves from M = 4096 to M = 8192 between these two window widths (nCorr = nDel + 100)
RANGE_SWITCH_4096_8192 = (3047, 3048)

CAF_ROWS = [
    # Doppler edges: nDop on both sides of every Bluestein length (M2 = 256 ... 16384)
    # (nCorr >= 20 keeps the largest lag, 17, inside a batch: the oracle's nfft-point correlation would alias it)
    _doppler_row(63, 64, 256), _doppler_row(64, 64, 512),
    _doppler_row(127, 40, 512), _doppler_row(128, 40, 1024),
    _doppler_row(255, 40, 1024), _doppler_row(256, 40, 2048),
    _doppler_row(511, 30, 2048), _doppler_row(512, 30, 4096),
    _doppler_row(1023, 20, 4096), _doppler_row(1024, 20, 8192),
    _doppler_row(2047, 20, 8192), _doppler_row(2048, 20, 16384),
    _doppler_row(4095, 20, 16384),                                  # 8191 bins: the largest accepted
    # delay edges: every range FFT length, the 4096 -> 8192 switch, and the widest windows
    _delay_row(257, 512), _delay_row(600, 1024), _delay_row(1000, 2048), _delay_row(3000, 4096),
    _delay_row(RANGE_SWITCH_4096_8192[0], 4096), _delay_row(RANGE_SWITCH_4096_8192[1], 8192),
    _delay_row(7168, 8192), _delay_row(8192, 8192),                 # 8192 bins: one new sample per segment
]

# rejected by the planner
CAF_REJECTED = [
    (-3, 17, -4096, 4096, 8193 * 12, 8193 * 12, True),              # 8193 Doppler bins
    (-10, 8193 - 11, -15, 15, 31 * 8293, 31 * 8293, True),          # 8193 delay bins
]


def row_id(row):
    return f"nDop{row['n_dop']}-nDel{row['n_del']}"


def plan_range_log2m(n_del, n_corr):
    """Restatement of plan_range (caf.cu) without environment overrides: log2 of the range FFT length."""
    best, best_l = 1e300, 0
    for l in range(8, 14):
        M = 1 << l
        L = M - n_del + 1
        if L < 1 or (L < M // 8 and l < 13):
            continue
        cost = (2.0 * ((n_corr + L - 1) // L) + 1.0) * M * l
        if l == 13:
            cost *= 1.15
        if l <= 10:
            cost *= 1.25
        if cost < best:
            best, best_l = cost, l
    return best_l


def default_kernels(M, M2):
    """The kernel templates the default environment runs for (M, M2) (caf.cu plan_range / caf_setup_device)."""
    rng = "caf_range_dit_kernel" if 512 <= M <= 4096 else "caf_range_kernel"
    dop = "caf_doppler_dit_kernel" if 512 <= M2 <= 4096 else "caf_doppler_kernel"
    return f"{rng}<{M.bit_length() - 1}>", f"{dop}<{M2.bit_length() - 1}>"


# ------------------------------------------------------------------------------------------ detection restatements
def cfar_1d(m, delay, doppler, noisePower, pfa, nGuard, nTrain, minDelay, minDoppler):
    """O.cfar_1d over the whole map at once.  The training cells are added one offset at a time in the reference's
    order (leading cells k > 0 only, then trailing cells), so every sum, threshold and decision is bit-identical."""
    nGuard, nTrain, minDelay = O._int8(nGuard), O._int8(nTrain), O._int8(minDelay)
    m = np.asarray(m, dtype=np.complex128)
    delay = np.asarray(delay)
    doppler = np.asarray(doppler, dtype=np.float64)
    nDop, nDel = m.shape
    sq = np.abs(m * m)
    j = np.arange(nDel)
    noise = np.zeros(m.shape)
    cells = np.zeros(nDel, dtype=np.int64)
    offsets = [(d, True) for d in range(-nGuard - nTrain, -nGuard)] + [(d, False) for d in range(nGuard + 1, nGuard + nTrain + 1)]
    for d, leading in offsets:
        k = j + d
        ok = (k > 0 if leading else k >= 0) & (k < nDel)
        shifted = np.zeros(m.shape)
        shifted[:, ok] = sq[:, k[ok]]
        noise = noise + shifted
        cells += ok
    alpha = np.array([n * (math.pow(pfa, -1.0 / n) - 1) if n else np.nan for n in range(int(cells.max(initial=0)) + 1)])
    with np.errstate(invalid="ignore", divide="ignore"):
        thr = alpha[cells] * (noise / np.where(cells > 0, cells, 1))
        det = (sq > thr) & (cells > 0)
        snr = 10.0 * np.log10(np.abs(m)) - noisePower
    det &= (delay >= minDelay)[None, :]
    det &= ~(np.abs(doppler) < minDoppler)[:, None]
    r, c = np.nonzero(det)                                  # row-major: the reference's emission order
    return (c + delay[0]).astype(np.float64), doppler[r].astype(np.float64), snr[r, c]


def centroid(delay, doppler, snr, nDelay, nDoppler, resolutionDoppler, chunk=1024):
    """O.centroid with the pairwise test done a block of rows at a time."""
    nDelay &= 0xFFFF
    nDoppler &= 0xFFFF
    delay, doppler, snr = (np.asarray(v, dtype=np.float64) for v in (delay, doppler, snr))
    n = snr.shape[0]
    keep = np.ones(n, dtype=bool)
    di = np.trunc(delay).astype(np.int64)
    dmin = ((di - nDelay) & 0xFFFF).astype(np.float64)
    dmax = ((di + nDelay) & 0xFFFF).astype(np.float64)
    fmin = doppler - (nDoppler * resolutionDoppler)
    fmax = doppler + (nDoppler * resolutionDoppler)
    for s in range(0, n, chunk):
        i = np.arange(s, min(n, s + chunk))
        near = ((delay[None, :] > dmin[i, None]) & (delay[None, :] < dmax[i, None]) &
                (doppler[None, :] > fmin[i, None]) & (doppler[None, :] < fmax[i, None]))
        near[np.arange(i.shape[0]), i] = False
        keep[i] = ~np.any(near & (snr[i, None] < snr[None, :]), axis=1)
    return delay[keep], doppler[keep], snr[keep]


def oracle_scene_map(seed):
    """The map, axes and noise power of the detection parity tests (tests/test_det_gpu.py): a 131 x 1001 map of a
    filtered two-target scene."""
    from blah2_b200.scene import make_scene, Target
    fs, n = 2000000, 200000
    geom = (-10, 120, -5000, 5000, fs, n, True)
    sc = make_scene(n, fs, seed=seed, targets=[Target(37, 3000.0, -30.0), Target(92, -2000.0, -35.0)])
    g = O.ambiguity_geometry(*geom)
    out = O.chain(sc.x, sc.y, g, clutter=(-10, 60))
    return g, out["map"], out["noisePower"]


# the parameter sets of test_det_gpu.test_cfar_edge_parameters
CFAR_PARAMS = [
    dict(pfa=1e-5, nGuard=2, nTrain=6, minDelay=5, minDoppler=15.0),
    dict(pfa=1e-12, nGuard=2, nTrain=6, minDelay=5, minDoppler=15.0),
    dict(pfa=1e-5, nGuard=2, nTrain=6, minDelay=5, minDoppler=1e9),
    dict(pfa=1e-5, nGuard=2, nTrain=0, minDelay=5, minDoppler=15.0),
    dict(pfa=1e-2, nGuard=1, nTrain=3, minDelay=-128, minDoppler=0.0),
    dict(pfa=1e-3, nGuard=258, nTrain=4, minDelay=300, minDoppler=0.0),
    dict(pfa=1e-3, nGuard=0, nTrain=1, minDelay=-128, minDoppler=0.0),    # the planted-spike setting of the GPU tests
]
