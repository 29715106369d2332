"""Case table shared by tests/test_spectrum_envelope_cpu.py and tests/test_spectrum_envelope_gpu.py.

The spectrum stage (blah2_b200/csrc/spectrum.cu) folds the first nfft = nSpectrum * decimation samples onto nSpectrum
columns, FOLD_UNROLL = 8 rows at a time in chunks of rows (two columns per thread when nSpectrum is even and the
float2 input starts 16-byte aligned), then takes an nSpectrum-point DFT whose phases are running products re-seeded
from a table every DFT_RESEED = 64 steps of a chain; a chain steps 128 bins, so re-seeding starts above 8192 bins.
The DFT stages g in shared memory up to 12288 bins (more than 48 KB of it above 3072) and reads it from global memory
beyond.  The rows below sit on both sides of each of those boundaries, at decimations below, at and just above the
fold's unroll, and at blah2's own n = 2e7, bandwidth 2000 (decimation 10^4, many fold chunks).

Each row is (n, bandwidth) with n = nSpectrum * decimation + extra, 0 <= extra < decimation: the input has samples
past nfft.  bandwidth = n / (decimation + 1/2) puts n / bandwidth half-way between two integers, so that
decimation = floor(n / bandwidth) does not depend on how the division rounds.
"""

# the kernel parameters the rows are laid against (spectrum.cu)
FOLD_UNROLL = 8
DFT_SMEM_48K = 3072        # nSpectrum * 16 B of staged g: at most 48 KB up to here
DFT_RESEED_FROM = 8192     # 64 running-product steps of 128 bins: chains longer than this re-seed
DFT_SMEM_MAX = 12288       # g in shared memory up to here, read from global memory above
MAX_BINS = 65536


def row(n_spectrum, dec, extra=0):
    assert 0 <= extra < dec
    n = n_spectrum * dec + extra
    return dict(n=n, bw=n / (dec + 0.5), n_spectrum=n_spectrum, dec=dec, nfft=n_spectrum * dec)


# (nSpectrum, decimation, extra)
ROWS = [row(*r) for r in [
    (1, 1, 0), (1, 17, 5), (2, 9, 3), (8, 7, 6), (8, 16, 0), (9, 8, 3),
    (3071, 2, 1), (3072, 8, 5), (3073, 9, 8), (3074, 1, 0),
    (8191, 15, 14), (8192, 16, 3), (8193, 7, 0), (8194, 2, 1),
    (12287, 1, 0), (12288, 17, 16), (12289, 8, 7), (12290, 15, 2),
    (65535, 2, 1), (65536, 1, 0), (65536, 9, 4),
]] + [dict(n=20000000, bw=2000.0, n_spectrum=2000, dec=10000, nfft=20000000)]   # blah2.cpp's bandwidth


def row_id(r):
    return f"bins{r['n_spectrum']}-dec{r['dec']}-n{r['n']}"
