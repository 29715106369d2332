"""CPU: every row of tests/spectrum_cases.py plans the geometry it was written for, and together the rows reach every
boundary of the spectrum kernels' plan (b200dd_spectrum_plan, no device needed)."""
import pytest

import spectrum_cases as S
from blah2_b200 import capi
from oracle import blah2_oracle as O


@pytest.mark.parametrize("r", S.ROWS, ids=S.row_id)
def test_row_geometry(r):
    g, freq = capi.spectrum_plan(r["n"], r["bw"])
    assert (g.decimation, g.n_spectrum, g.nfft) == (r["dec"], r["n_spectrum"], r["nfft"])
    assert (g.decimation, g.n_spectrum, g.nfft) == O.spectrum_geometry(r["n"], r["bw"])
    assert r["nfft"] <= r["n"] < r["nfft"] + r["dec"]
    # the fold's chunking covers every row of the input exactly once
    assert g.fold_rows_per_chunk >= S.FOLD_UNROLL
    assert (g.fold_chunks - 1) * g.fold_rows_per_chunk < g.decimation <= g.fold_chunks * g.fold_rows_per_chunk
    assert freq.shape == (0,)


def test_rows_reach_every_boundary():
    plans = [capi.spectrum_plan(r["n"], r["bw"])[0] for r in S.ROWS]
    bins = {int(g.n_spectrum) for g in plans}
    decs = {int(g.decimation) for g in plans}
    assert {1, 2, 8} <= bins and S.MAX_BINS in bins
    for edge in (S.DFT_SMEM_48K, S.DFT_RESEED_FROM, S.DFT_SMEM_MAX):
        below = {b for b in bins if b <= edge and b > edge - 8}
        above = {b for b in bins if b > edge and b <= edge + 8}
        for side in (below, above):
            assert {b % 2 for b in side} == {0, 1}, (edge, side)
    assert {1, 2, 7, 8, 9, 15, 16, 17} <= decs
    assert any(d >= 10000 for d in decs)
    # a decimation below the unroll, a multiple of it and one with a tail, each with an even bin count (the
    # two-column fold) and an odd one (the one-column fold)
    for pred in (lambda d: d < S.FOLD_UNROLL, lambda d: d % S.FOLD_UNROLL == 0, lambda d: d % S.FOLD_UNROLL != 0 and d > S.FOLD_UNROLL):
        assert {int(g.n_spectrum) % 2 for g in plans if pred(int(g.decimation))} == {0, 1}
    # a fold chunk whose last rows are fewer than the unroll
    assert any(int(g.decimation) % int(g.fold_rows_per_chunk) % S.FOLD_UNROLL for g in plans)
    # many fold chunks
    assert max(int(g.fold_chunks) for g in plans) >= 64
    # samples past nfft on most rows
    assert sum(r["n"] > r["nfft"] for r in S.ROWS) >= len(S.ROWS) // 2
