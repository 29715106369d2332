"""Synthetic passive-radar IQ scenes and the reference's replay file format.

Seeded generator used by tests and bench.py (SURVEY.md s8(d)): reference channel x is an
int16-quantised complex Gaussian (the RSPduo replay range, reference
src/capture/rspduo/RspDuo.cpp:155-174); surveillance y is the direct path + static
clutter taps + a few moving targets + receiver noise, quantised to int16 as well.  All
values are exactly representable in float32, which is the device IQ format.

``write_rspduo`` / ``read_rspduo`` implement the reference's replay layout: little-endian
int16 ``I1 Q1 I2 Q2`` per time instant (reader at
test/unit/process/ambiguity/TestAmbiguity.cpp:39-69).  ``iq_from_ci8`` / ``iq_from_cf32`` state the samples blah2
takes from its HackRF / Kraken (int8) and USRP (complex float32) sources.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np


@dataclass
class Target:
    delay: int  # bins
    doppler: float  # Hz
    gain_db: float  # relative to the reference channel amplitude


@dataclass
class Scene:
    x: np.ndarray  # complex128, integer valued
    y: np.ndarray
    targets: list = field(default_factory=list)


def make_scene(n: int, fs: float, seed: int = 20260923, targets=None, n_clutter: int = 16, direct_gain: float = 0.5,
               sigma_ref: float = 1500.0, sigma_noise: float = 20.0, quantise: bool = True) -> Scene:
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * (sigma_ref / np.sqrt(2.0))
    if quantise:
        x = np.clip(np.round(x.real), -32767, 32767) + 1j * np.clip(np.round(x.imag), -32767, 32767)
    if targets is None:
        targets = [Target(37, 55.0, -50.0), Target(92, -103.0, -55.0), Target(151, 78.0, -60.0),
                   Target(230, -41.0, -58.0)]
    y = direct_gain * x
    # static clutter: taps at delays 1..n_clutter-1 falling from -10 dB to -40 dB (delay 0 is the direct path)
    for d in range(1, n_clutter):
        g_db = -10.0 - 30.0 * (d - 1) / max(1, n_clutter - 2)
        ph = np.exp(1j * rng.uniform(0, 2 * np.pi))
        tap = (10.0 ** (g_db / 20.0)) * ph
        y[d:] += tap * x[:-d]
    t = np.arange(n, dtype=np.float64) / float(fs)
    for tg in targets:
        a = 10.0 ** (tg.gain_db / 20.0)
        shifted = np.zeros(n, dtype=np.complex128)
        if tg.delay > 0:
            shifted[tg.delay:] = x[: n - tg.delay]
        else:
            shifted[:] = x
        y = y + a * shifted * np.exp(2j * np.pi * tg.doppler * t)
    y = y + (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * (sigma_noise / np.sqrt(2.0))
    if quantise:
        y = np.clip(np.round(y.real), -32767, 32767) + 1j * np.clip(np.round(y.imag), -32767, 32767)
    return Scene(np.asarray(x, dtype=np.complex128), np.asarray(y, dtype=np.complex128), list(targets))


def random_iq(n: int, seed: int, lo: float = -100.0, hi: float = 100.0):
    """The reference unit test's input style (uniform(-100,100) I and Q,
    TestAmbiguity.cpp:24-32) but SEEDED."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(lo, hi, n) + 1j * rng.uniform(lo, hi, n)
    y = rng.uniform(lo, hi, n) + 1j * rng.uniform(lo, hi, n)
    return x, y


def write_rspduo(path: str, x: np.ndarray, y: np.ndarray) -> None:
    n = x.shape[0]
    buf = np.empty((n, 4), dtype="<i2")
    buf[:, 0] = np.clip(np.round(x.real), -32768, 32767)
    buf[:, 1] = np.clip(np.round(x.imag), -32768, 32767)
    buf[:, 2] = np.clip(np.round(y.real), -32768, 32767)
    buf[:, 3] = np.clip(np.round(y.imag), -32768, 32767)
    buf.tofile(path)


def _complex(re: np.ndarray, im: np.ndarray) -> np.ndarray:
    out = np.empty(re.shape[0], dtype=np.complex128)
    out.real, out.imag = re, im  # not re + 1j * im, which loses the sign of a -0.0 imaginary part
    return out


def iq_from_ci8(buf) -> np.ndarray:
    """The complex128 samples blah2 pushes into IqData from one channel's int8 I/Q buffer: every byte read as int8_t
    and widened to double.  HackRF hands over int8 (src/capture/hackrf/HackRf.cpp:116-128); Kraken reads rtl-sdr's
    offset-binary bytes through an int8_t pointer (src/capture/kraken/Kraken.cpp:97-112), so 0x80 becomes -128."""
    b = np.ascontiguousarray(buf).view(np.int8).reshape(-1, 2).astype(np.float64)
    return _complex(b[:, 0], b[:, 1])


def iq_from_cf32(buf) -> np.ndarray:
    """The complex128 samples blah2 pushes into IqData from one channel's UHD fc32 buffer
    (src/capture/usrp/Usrp.cpp:54-91): each float widened to double."""
    f = np.ascontiguousarray(buf).view(np.float32).reshape(-1, 2).astype(np.float64)
    return _complex(f[:, 0], f[:, 1])


def read_rspduo(path: str, n: int | None = None):
    raw = np.fromfile(path, dtype="<i2")
    raw = raw[: (raw.shape[0] // 4) * 4].reshape(-1, 4)
    if n is not None:
        raw = raw[:n]
    x = raw[:, 0].astype(np.float64) + 1j * raw[:, 1].astype(np.float64)
    y = raw[:, 2].astype(np.float64) + 1j * raw[:, 3].astype(np.float64)
    return x, y
