"""The reference build of the class harness (oracle/dropinclass/class_capi.cpp with blah2's own classes) against the
oracle and det_cases' restatement, on the sequences tests/test_dropin_classes_gpu.py gives both builds: one object
over many calls, as blah2.cpp keeps its objects.  This pins the oracle to the reference for these lifecycles.
Skipped where the reference build is absent (it is built from the blah2 sources)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import det_cases as D  # noqa: E402
import dropin_class_cases as K  # noqa: E402
import spectrum_cases as S  # noqa: E402

from oracle import blah2_oracle as O  # noqa: E402
from oracle import dropin_class as DC  # noqa: E402

pytestmark = pytest.mark.skipif(not DC.available("ref"), reason="reference class harness not built")

SMALL_ROWS = [r for r in S.ROWS if r["n"] <= 1 << 18]


@pytest.fixture(scope="module")
def maps():
    return [dict(name=n, map=m, delay=dl, doppler=dp, noise=z, sq=D.sq_values(m),
                 db=K.cpu_db(m, z)) for n, m, dl, dp, z in K.map_sequence()]


def test_spectrum_analyser_over_consecutive_fifos():
    rng = np.random.default_rng(5)
    for r in SMALL_ROWS:
        sa = DC.SpectrumAnalyserClass("ref", r["n"], r["bw"])
        for _ in range(2):
            x = rng.standard_normal(r["n"]) + 1j * rng.standard_normal(r["n"])
            s, f, left = sa.process(x)
            want, freq = O.spectrum_process(x, r["n"], r["bw"])
            assert left == r["n"] and f.size == freq.size == 0
            assert float(np.max(np.abs(s - want))) <= 1e-11 * float(np.max(np.abs(want))), S.row_id(r)
        sa.close()


@pytest.mark.parametrize("params", K.CFAR_PARAMS, ids=K.CFAR_IDS)
def test_cfar_object_is_the_restatement(maps, params):
    o = DC.CfarClass("ref", *params)
    for c in maps:
        got = o.process(c["map"], c["delay"], c["doppler"], c["noise"])
        assert D.same(got, D.cfar(c["sq"], c["db"], c["delay"], c["doppler"], *params)), c["name"]
    o.close()


def test_centroid_object_is_the_restatement():
    P = K.CENTROID_P
    o = DC.CentroidClass("ref", P["nDelay"], P["nDoppler"], P["res"])
    for name, d, f, s in K.centroid_sequence():
        if d.size <= 4096:
            assert D.same(o.process(d, f, s), D.centroid(d, f, s, P["nDelay"], P["nDoppler"], P["res"])), name
    o.close()


@pytest.mark.parametrize("flags", [(True, True), (True, False), (False, True), (False, False)])
def test_interpolate_object_is_the_restatement(maps, flags):
    o = DC.InterpolateClass("ref", *flags)
    for c in maps:
        if c["map"].shape[0] < 2 or c["map"].shape[1] < 3:
            continue
        lst = D.centroid(*D.cfar(c["sq"], c["db"], c["delay"], c["doppler"], D.PFA, 1, 4, -128, 0.0), 2, 2, 10.0)
        keep = ~D.interpolate(*lst, c["db"], c["delay"], c["doppler"], True, True)[3]
        lst = tuple(a[keep] for a in lst)
        got = o.process(*lst, c["map"], c["delay"], c["doppler"], c["noise"])
        assert D.same(got, D.interpolate(*lst, c["db"], c["delay"], c["doppler"], *flags)[:3]), c["name"]
    o.close()


@pytest.mark.parametrize("clutter", [True, False], ids=["clutter", "no_clutter"])
@pytest.mark.parametrize("window", sorted(K.PAIR_GEOMS))
def test_fifo_pair_follows_the_oracle(window, clutter, relerr):
    """After every CPI: the map is the oracle's map of the queued samples, get_n_samples() is nDop * nCorr, and the
    samples left in x are the queue rotated by the phase of each sample's position in it before the CPI."""
    geom = K.PAIR_GEOMS[window]
    o = DC.PairClass("ref", *geom, K.PAIR_CLUTTER if clutter else None, K.PAIR_FIFO)
    g = O.ambiguity_geometry(*geom)
    for k, (x, y) in enumerate(K.pair_pushes(g.n_used, g.n)):
        o.push(x, y)
        if clutter:
            assert o.filter() == (k != K.PAIR_FAIL_AT), k
        qx, qy = o.fifo(0), o.fifo(1)
        m = o.ambiguity((g.nDopplerBins, g.nDelayBins))
        assert o.n_samples() == g.n_used
        want, lx, ly = O.ambiguity_process(qx, qy, g)
        if k == K.PAIR_FAIL_AT:
            assert not np.any(m)
        else:
            assert max(relerr(m, want)) < 1e-9, k
        left, rot = o.fifo(0), O.ambiguity_prerotate(qx, g)[g.n_used:]
        assert (left.size, o.fifo(1).size) == (lx, ly), k
        assert float(np.max(np.abs(left - rot), initial=0.0)) <= 1e-12 * float(np.max(np.abs(qx))), k
    o.close()
