"""Inputs of the max-hold fixture (tests/golden/maxhold_docs.npz): sequences of CPI maps, generated instead of stored.

Each sequence has the shape, sample rate and axes of one map of tests/map_json_maps.py and N_SEQ CPIs, three more
than the window of 20, so the window wraps.  CPI i's map is hash_map with its own seed.  The "medium" sequence
has a CPI with one zero cell: it has no map document, and the fixture's windows leave it out.
"""
from __future__ import annotations

import numpy as np

from map_json_maps import MAPS, hash_map

N_SEQ = 23

# name -> map spec of map_json_maps.MAPS plus the first timestamp and its step per CPI; "zero_cpi": the CPI with a
# zero cell.  Timestamps cover 0, 2^53 + 1 and 2^64 - 1, which JSON.parse rounds.
SEQS = {
    "tiny": dict(MAPS["tiny"], ts=0, ts_step=1),
    "small": dict(MAPS["small"], ts=2 ** 64 - 1, ts_step=-1),
    "medium": dict(MAPS["medium"], ts=2 ** 53 + 1, ts_step=1000, zero_cpi=9),
    "cfg2": dict(MAPS["cfg2"], ts_step=1000),
    "cfg3": dict(MAPS["cfg3"], ts_step=1000),
    "cfg5": dict(MAPS["cfg5"], ts_step=1000),
}


def timestamp(spec, i: int) -> int:
    return spec["ts"] + spec["ts_step"] * i


def zero_cell(spec):
    """(row, column) of the zero cell of the "zero_cpi" CPI."""
    return spec["nDop"] // 3, spec["nDel"] // 2


def seq_map(spec, i: int, with_zero: bool = True):
    """(map complex128 [nDop, nDel], delay, doppler) of CPI i; with_zero=False gives the zero-cell CPI's map before
    its cell is zeroed (whose set_metrics values the fixture stores)."""
    m, delay, doppler = hash_map(dict(spec, seed=spec["seed"] * 64 + i))
    if with_zero and spec.get("zero_cpi") == i:
        m[zero_cell(spec)] = 0.0
    return m, delay, doppler
