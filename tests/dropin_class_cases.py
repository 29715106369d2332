"""Input sequences shared by tests/test_dropin_classes_cpu.py and tests/test_dropin_classes_gpu.py: maps whose shape
grows, shrinks, changes aspect and grows again for one CfarDetector1D or Interpolate object, detection lists for one
Centroid object, and the samples pushed into one FIFO pair over consecutive CPIs for Ambiguity and WienerHopf.

Map shapes (nDop x nDel) in order, with the handle a reused drop-in object must hold for each:
  scene 201 x 66 -> ties 17 x 48 (smaller) -> scene 401 x 20 (more rows, fewer cells) -> window-edge ties of widths
  1 .. 20 (smaller) -> scene 41 x 131 (wider, fewer rows) -> scene 201 x 66 again -> spikes of 2049 detections.
"""
from __future__ import annotations

import functools

import numpy as np

import det_cases as D
from blah2_b200.scene import Target, make_scene
from oracle import blah2_oracle as O

# (delayMin, delayMax, dopplerMin, dopplerMax, fs, n): Doppler resolution fs / n = 5 Hz
SCENE_GEOMS = {"a": (-5, 60, -500, 500, 200000, 40000), "tall": (-2, 17, -1000, 1000, 200000, 40000),
               "wide": (-10, 120, -100, 100, 200000, 40000)}
SCENE_NOISE_SEED = {"a": 11, "tall": 12, "wide": 13}


@functools.lru_cache(maxsize=None)
def scene_map(name):
    """The oracle's map of a scene with two targets, its axes and its set_metrics noise power."""
    g = O.ambiguity_geometry(*SCENE_GEOMS[name], True)
    sc = make_scene(g.n, g.fs, seed=SCENE_NOISE_SEED[name],
                    targets=[Target(7, 300.0, -25.0), Target(15, -200.0, -28.0)])
    m, _, _ = O.ambiguity_process(sc.x, sc.y, g)
    noise, _ = O.set_metrics(m)
    return m, np.asarray(g.delay, np.int32), np.asarray(g.doppler, np.float64), float(noise)


def map_sequence():
    """[(name, map, delay, doppler, noisePower)] in the order of the module docstring."""
    seq = [("scene_a",) + scene_map("a")]
    cases = {c["name"]: c for c in D.cfar_cases()}
    c = cases["f32_ties"]
    seq.append(("f32_ties", c["map"], c["delay"], c["doppler"], D.NOISE))
    seq.append(("scene_tall",) + scene_map("tall"))
    for w in range(1, 21):
        c = cases[f"edges_w{w}"]
        seq.append((c["name"], c["map"], c["delay"], c["doppler"], D.NOISE))
    c = cases["mixed_windows"]
    seq.append((c["name"], c["map"], c["delay"], c["doppler"], D.NOISE))
    seq.append(("scene_wide",) + scene_map("wide"))
    seq.append(("scene_a_again",) + scene_map("a"))
    m, delay, doppler = D.spike_map(2049)
    seq.append(("spikes_2049", m, delay, doppler, D.NOISE))
    return seq


# (pfa, nGuard, nTrain, minDelay, minDoppler) as given to the constructor, before its int8_t narrowing
CFAR_PARAMS = [
    (1e-4, 2, 6, 3, 15.0),            # smoke()'s detector
    (D.PFA, 258, 264, 261, 15.0),     # narrowed to 2, 8, 5
    (D.PFA, 1, 8, -128, 0.0),         # minDelay at the int8 minimum, up to 16 training cells
    (D.PFA, 0, 16, 127, 0.0),         # minDelay at the int8 maximum, up to 32 training cells
    (1e-3, 0, 0, -128, 0.0),          # no training cells: alpha is NaN, nothing is detected
    (1e-3, 3, 1, 0, 1e300),           # every row below minDoppler
    (D.PFA, 2, 255, 0, 15.0),         # nTrain narrowed to -1: no training cells
]
CFAR_IDS = ["smoke", "int8_narrowing", "min_delay_int8_min", "min_delay_int8_max", "no_training", "no_rows",
            "negative_train"]

CENTROID_P = D.CENTROID_PARAMS


def cpu_db(m, noise):
    """Every cell's 10 log10|z| - noise as the reference computes it: |z| is glibc's hypot (std::abs of a complex;
    numpy's abs of a complex can differ from it in the last place), log10 glibc's."""
    m = np.asarray(m, np.complex128)
    return D.db_values(D.log10_abs(np.hypot(m.real, m.imag)), noise)


def clustered_list(n, n_peaks=64, seed=3):
    """n detections in n_peaks clusters: each cluster's peak first in the list (so the reference's pairwise search
    stops within the first n_peaks entries for every other detection), the rest of the cluster within (nDelay - 1)
    cells and two Doppler resolution steps of its peak, at lower or equal SNRs."""
    rng = np.random.default_rng(seed)
    nD, res = CENTROID_P["nDelay"], CENTROID_P["res"]
    pd = 100.0 + 20.0 * np.arange(n_peaks)
    pf = np.round(rng.uniform(-20, 20, n_peaks), 1)
    ps = 50.0 + rng.integers(0, 5, n_peaks)
    k = rng.integers(0, n_peaks, n - n_peaks)
    d = pd[k] + rng.integers(-(nD - 1), nD, n - n_peaks)
    f = pf[k] + res * rng.integers(-2, 3, n - n_peaks)
    s = np.minimum(ps[k] - rng.integers(0, 30, n - n_peaks), ps[k])
    return np.concatenate([pd, d]), np.concatenate([pf, f]), np.concatenate([ps, s]).astype(np.float64)


def centroid_sequence():
    """[(name, delay, doppler, snr)]: every list of det_cases.centroid_cases(), then one longer than 512 * 512 / 2
    and one of exactly 2^18 detections."""
    seq = list(D.centroid_cases())
    for n in (512 * 512 // 2 + 1, 1 << 18):
        seq.append((f"clusters_{n}",) + clustered_list(n))
    return seq


# ---------------------------------------------------------------------------------------------- FIFO pair
PAIR_GEOMS = {"symmetric": (0, 31, -40, 40, 10000, 5000, True), "off_centre": (0, 31, -20, 60, 10000, 5000, True)}
PAIR_CLUTTER = (-2, 10)
PAIR_FIFO = 5040     # more than n = 5000, so WienerHopf sees a FIFO longer than its nSamples
PAIR_CPIS = 25
PAIR_FAIL_AT = 12    # the CPI whose reference channel is all zeros


def pair_pushes(n_used, n, seed=7):
    """Per CPI, the (x, y) pushed before it: n samples first, then n_used + 3, so 3 more samples carry over each CPI
    and the FIFOs reach their capacity; at PAIR_FAIL_AT x is PAIR_FIFO zeros, which flush it."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(PAIR_CPIS):
        m = n if k == 0 else n_used + 3
        x = (rng.standard_normal(m) + 1j * rng.standard_normal(m)) * 100.0
        y = (rng.standard_normal(m) + 1j * rng.standard_normal(m)) * 30.0 + 0.5 * np.roll(x, 3)
        if k == PAIR_FAIL_AT:
            x = np.zeros(PAIR_FIFO, dtype=np.complex128)
        out.append((x, y))
    return out
