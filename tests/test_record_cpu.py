"""CPU: CPI records without a GPU -- argument checks of the export / import entry points, the record-size formula,
and the independent-CPI plan at world 2 and 3 on gloo with stand-in records tagged by CPI index."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from blah2_b200 import capi
from blah2_b200.process import record_bytes


def test_null_arguments_are_rejected():
    lib = capi.load()
    nb = C.c_size_t(7)
    assert lib.b200dd_pipeline_enable_export(None, 4096, C.byref(nb)) == capi.ERR_ARG
    assert nb.value == 0
    assert lib.b200dd_pipeline_enable_export(None, 4096, None) == capi.ERR_ARG
    rec = C.c_void_p(1)
    assert lib.b200dd_pipeline_export_record(None, C.byref(rec)) == capi.ERR_ARG
    assert rec.value is None
    assert lib.b200dd_pipeline_export_record(None, None) == capi.ERR_ARG
    assert lib.b200dd_pipeline_submit_record(None, None, None) == capi.ERR_ARG
    assert lib.b200dd_pipeline_submit_record(None, C.c_void_p(16), C.c_void_p(16)) == capi.ERR_ARG


@pytest.mark.parametrize("max_detections", [0, (1 << 18) + 1, 0xFFFFFFFF])
def test_max_detections_out_of_range_is_rejected(max_detections):
    lib = capi.load()
    nb = C.c_size_t()
    assert lib.b200dd_pipeline_enable_export(None, max_detections, C.byref(nb)) == capi.ERR_ARG
    assert "max_detections" in capi.last_error()


def test_max_detections_in_range_reaches_the_handle_check():
    lib = capi.load()
    for m in (1, 4096, 1 << 18):
        assert lib.b200dd_pipeline_enable_export(None, m, None) == capi.ERR_ARG
        assert "null handle" in capi.last_error()


def test_record_size_formula():
    assert record_bytes(4096) == 64 + 24 * 4096                 # 96 KB of slots next to the header
    assert record_bytes(4096, detection=False) == 64
    assert record_bytes(1) == 96                                 # 64 + 24, rounded up to 16
    assert record_bytes(3, timing=True) == 64 + 80 + 80          # 72 rounded up to 80
    assert record_bytes(4096, n_spectrum=1000, timing=True) == 64 + 80 + 16000 + 24 * 4096
    assert record_bytes(1 << 18, n_spectrum=2000, timing=True) == 64 + 80 + 32000 + 24 * (1 << 18)
    for m in (1, 2, 5, 4095, 4096):
        for ns in (0, 1, 7):
            for t in (False, True):
                for d in (False, True):
                    b = record_bytes(m, ns, t, d)
                    assert b % 16 == 0 and 0 <= b - (64 + 80 * t + 16 * ns + 24 * m * d) < 16


# ---- the independent-CPI plan on gloo ------------------------------------------------------------------------------
_RB = 40          # stand-in record bytes
_MAP = (3, 5)


def _record_of(c):
    r = torch.zeros(_RB, dtype=torch.uint8)
    r[:8] = torch.from_numpy(np.array([c], dtype=np.int64).view(np.uint8))
    r[8:] = c % 251
    return r


def _worker(rank, world, port, n_cpis, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from blah2_b200.shard import IndependentCpiPlan, TorchComm, cpi_indices
        plan = IndependentCpiPlan(TorchComm(rank, world), _RB, _MAP, "cpu", depth=2)
        computed, got = [], []

        def compute(c):
            computed.append(c)
            return _record_of(c), torch.full(_MAP, complex(c, -2 * c), dtype=torch.complex64)

        def consume(c, record, m):
            tag = int(record[:8].numpy().copy().view(np.int64)[0])
            got.append((c, tag, bool(torch.equal(record, _record_of(c))), m.numpy().copy()))

        plan.run(n_cpis, compute, consume)
        assert computed == cpi_indices(n_cpis, rank, world)
        if rank == 0:
            q.put(got)
        else:
            assert got == []
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,n_cpis", [(2, 5), (2, 6), (3, 7), (3, 2)])
def test_independent_cpi_plan_gloo(world, n_cpis):
    """Rank 0 consumes every CPI exactly once, in CPI order, each with its own record and its own map."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + (os.getpid() % 2000) + 10 * world + n_cpis
    procs = [ctx.Process(target=_worker, args=(r, world, port, n_cpis, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = q.get(timeout=240)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert [c for c, _, _, _ in got] == list(range(n_cpis))
    for c, tag, same, m in got:
        assert tag == c and same
        assert m.shape == _MAP and np.all(m == complex(c, -2 * c))
