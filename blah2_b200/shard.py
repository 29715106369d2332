"""Multi-GPU sharding of the hot path: independent CPIs round-robin over ranks.

The path has no exchange step between CPIs (BASELINE config 4: "stream of independent CPIs sharded
round-robin"), so the data path needs no collective; the only communication is the final gather of
the finished maps to rank 0 (NCCL over NVLink on GPUs, gloo in the CPU tests).  One process per GPU.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from .capi import STAMP_CHAIN, STAMP_CLUTTER, STAMP_SPECTRUM
from .process import _Handle


class Comm(_Handle):
    """The C-ABI communicator (include/b200dd.h b200dd_comm_*: NCCL issued from C on its own stream).

    One per process / GPU.  The 128-byte NCCL id is created on rank 0 and handed to the other ranks through
    torch.distributed's default process group (any backend) -- plumbing; the data path below never touches torch.
    """
    _destroy = "b200dd_comm_destroy"

    def __init__(self, rank: int, world: int, device: int):
        from . import capi
        self._capi = capi
        self._lib = capi.load()
        ident = np.zeros(128, dtype=np.uint8)
        if rank == 0:
            capi.check(self._lib.b200dd_comm_get_unique_id(capi.ptr(ident)))
        if world > 1:
            t = torch.from_numpy(ident)
            if dist.get_backend() == "nccl":
                t = t.cuda(device)
            dist.broadcast(t, src=0)
            ident = t.cpu().numpy().copy()
        h = C.c_void_p()
        capi.check(self._lib.b200dd_comm_create(int(rank), int(world), capi.ptr(ident), int(device), C.byref(h)))
        self._h, self.rank, self.world = h, rank, world

    @staticmethod
    def _sp(stream):
        if stream is None:
            return None
        return C.c_void_p(stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream))

    def gather_async(self, send: torch.Tensor, recv, dst: int = 0, after=None):
        """Every rank's `send` (same byte size) lands on rank dst at recv[r]; returns at once."""
        nbytes = send.numel() * send.element_size()
        self._capi.check(self._lib.b200dd_comm_gather_async(self._h, self._capi.ptr(send),
                                                            self._capi.ptr(recv) if recv is not None else None,
                                                            nbytes, int(dst), self._sp(after)))

    def gatherv_async(self, send: torch.Tensor, recv, sizes, offsets, dst: int = 0, after=None):
        nbytes = send.numel() * send.element_size()
        sz = (C.c_size_t * self.world)(*[int(v) for v in sizes])
        of = (C.c_size_t * self.world)(*[int(v) for v in offsets])
        self._capi.check(self._lib.b200dd_comm_gatherv_async(self._h, self._capi.ptr(send), nbytes,
                                                             self._capi.ptr(recv) if recv is not None else None,
                                                             sz, of, int(dst), self._sp(after)))

    def allgatherv_async(self, send: torch.Tensor, recv: torch.Tensor, sizes, offsets, after=None):
        sz = (C.c_size_t * self.world)(*[int(v) for v in sizes])
        of = (C.c_size_t * self.world)(*[int(v) for v in offsets])
        self._capi.check(self._lib.b200dd_comm_allgatherv_async(self._h, self._capi.ptr(send), self._capi.ptr(recv), sz, of,
                                                                self._sp(after)))

    def allreduce_f64_async(self, buf: torch.Tensor, after=None):
        count = buf.numel() * (2 if buf.is_complex() else 1)
        self._capi.check(self._lib.b200dd_comm_allreduce_f64_async(self._h, self._capi.ptr(buf), count, self._sp(after)))

    def sendrecv_async(self, send, send_peer: int, recv, recv_peer: int, after=None):
        """One send (to send_peer) and / or one receive (from recv_peer) in one group; a peer of -1 skips that half."""
        sb = send.numel() * send.element_size() if (send is not None and send_peer >= 0) else 0
        rb = recv.numel() * recv.element_size() if (recv is not None and recv_peer >= 0) else 0
        self._capi.check(self._lib.b200dd_comm_sendrecv_async(self._h, self._capi.ptr(send) if sb else None, sb, int(send_peer),
                                                              self._capi.ptr(recv) if rb else None, rb, int(recv_peer),
                                                              self._sp(after)))

    def wait_stream(self, stream):
        """The communicator's stream waits for everything enqueued so far on `stream`."""
        self._capi.check(self._lib.b200dd_comm_wait_stream(self._h, self._sp(stream)))

    def join(self, stream):
        """`stream` waits for everything enqueued on the communicator so far."""
        self._capi.check(self._lib.b200dd_comm_join(self._h, self._sp(stream)))

    def torch_stream(self):
        """The communicator's CUDA stream as a torch stream (to record / wait on events for finer-grained ordering
        than join(): e.g. 'the gather that read THIS buffer has finished')."""
        if getattr(self, "_ts", None) is None:
            self._ts = torch.cuda.ExternalStream(int(self._lib.b200dd_comm_stream(self._h)))
        return self._ts

    def sync(self):
        self._capi.check(self._lib.b200dd_comm_sync(self._h))


def cpi_indices(n_cpis: int, rank: int, world: int) -> list[int]:
    """CPI c is processed by rank c mod world."""
    return list(range(rank, n_cpis, world))


def gather_maps(local_maps: torch.Tensor, n_cpis: int, rank: int, world: int, dst: int = 0):
    """local_maps: [k_r, nDop, nDel] complex64, the maps of cpi_indices(n_cpis, rank, world) in order.
    Returns on ``dst`` a tensor [n_cpis, nDop, nDel] in CPI order, None elsewhere."""
    if world == 1:
        return local_maps
    k_max = (n_cpis + world - 1) // world
    shape = tuple(local_maps.shape[1:])
    buf = torch.zeros((k_max,) + shape, dtype=local_maps.dtype, device=local_maps.device)
    buf[: local_maps.shape[0]] = local_maps
    flat = torch.view_as_real(buf).contiguous()   # gloo has no complex support; NCCL does not care
    gathered = [torch.empty_like(flat) for _ in range(world)] if rank == dst else None
    dist.gather(flat, gathered, dst=dst)
    if rank != dst:
        return None
    out = torch.empty((n_cpis,) + shape, dtype=local_maps.dtype, device=local_maps.device)
    for r in range(world):
        idx = cpi_indices(n_cpis, r, world)
        out[idx] = torch.view_as_complex(gathered[r])[: len(idx)]
    return out


class IndependentCpiPlan:
    """Independent CPIs over the ranks with every product on rank ``dst`` (BASELINE config 4).

    Rank r computes the CPIs c = r, r + world, ... (cpi_indices); each CPI's record (Pipeline.export_record) and map
    travel to ``dst`` in one round of two gathers per ``world`` CPIs (``comm.gather_async``), and ``dst`` hands them to
    ``consume`` in CPI order, c = 0, 1, 2, ..., which submits them to its importing pipeline(s)
    (Pipeline.submit_record) and fetches.  ``comm`` is a Comm on GPUs, a TorchComm in the CPU tests.

    Receive buffers form a ring of ``depth`` rounds: a round's buffers are gathered into again ``depth`` rounds later,
    so by then every CPI consumed from them must have been fetched (fetch() ends a CPI's reads of its map).  Importers
    that keep CPIs unfetched across rounds (a share set) need a deeper ring."""

    def __init__(self, comm, record_bytes: int, map_shape, device, depth: int = 1, dst: int = 0):
        self.comm, self.dst, self.depth = comm, dst, int(depth)
        shape = tuple(map_shape)
        # what a rank without a CPI in the last round sends: the gathers are collective
        self.pad_record = torch.zeros(int(record_bytes), dtype=torch.uint8, device=device)
        self.pad_map = torch.zeros(shape, dtype=torch.complex64, device=device)
        self.recv_record = self.recv_map = None
        if comm.rank == dst:
            self.recv_record = torch.empty((self.depth, comm.world, int(record_bytes)), dtype=torch.uint8, device=device)
            self.recv_map = torch.empty((self.depth, comm.world) + shape, dtype=torch.complex64, device=device)

    def run(self, n_cpis: int, compute, consume, after=None):
        """CPIs 0 .. n_cpis - 1.  On every rank, ``compute(c)`` enqueues CPI c on the stream ``after`` (None: the
        caller's ordering is synchronous) and returns its (record, map) tensors; the next round's compute is enqueued
        after this round's gathers have read them.  On ``dst``, ``consume(c, record, map)`` gets every CPI in order,
        its buffers complete."""
        comm, rank, world, dst = self.comm, self.comm.rank, self.comm.world, self.dst
        for k in range((n_cpis + world - 1) // world):
            # the last round's gathers have read what compute overwrites
            comm.join(after) if after is not None else comm.sync()
            c = k * world + rank
            record, m = compute(c) if c < n_cpis else (self.pad_record, self.pad_map)
            s = k % self.depth
            root = rank == dst
            comm.gather_async(record, self.recv_record[s] if root else None, dst, after=after)
            comm.gather_async(m, self.recv_map[s] if root else None, dst, after=None)
            if not root:
                continue
            comm.sync()                             # submit_record reads each record's header on the host
            for r in range(world):
                if k * world + r < n_cpis:
                    consume(k * world + r, self.recv_record[s, r], self.recv_map[s, r])


# ------------------------------------------------------------------------------------------
# ONE large CPI split over the ranks (BASELINE config 5)
# ------------------------------------------------------------------------------------------
def block_range(n: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous block [start, start+count) of n items for `rank` (sizes differ by at most one)."""
    base, rem = divmod(n, world)
    start = rank * base + min(rank, rem)
    return start, base + (1 if rank < rem else 0)


def _all_gather_rows(local: torch.Tensor, counts: list[int], world: int) -> torch.Tensor:
    """Concatenate row blocks of different heights from every rank (padded all_gather)."""
    k_max = max(counts)
    shape = tuple(local.shape[1:])
    buf = torch.zeros((k_max,) + shape, dtype=local.dtype, device=local.device)
    buf[: local.shape[0]] = local
    flat = torch.view_as_real(buf).contiguous()
    parts = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(parts, flat)
    return torch.cat([torch.view_as_complex(parts[r])[: counts[r]] for r in range(world)], dim=0)


def caf_single_cpi_sharded(amb, d_x_local: torch.Tensor, d_y_local: torch.Tensor, rank: int, world: int,
                           stream=None, dst: int = 0):
    """Cross-ambiguity function of ONE CPI whose IQ is spread over the ranks.

    The range stage is independent per batch, so rank r correlates the contiguous block of batches
    ``block_range(nDopplerBins, r, world)`` -- a contiguous 1/world slice of the IQ, which is all it
    holds (``d_x_local``, ``d_y_local``: complex64 CUDA tensors of that many batches * nCorr samples).
    The Doppler stage needs every batch of a delay column, hence ONE exchange: an all-gather of the
    range matrix (nDop x nDel complex64, <= 17 MB).  Each rank then transforms its tile of delay columns
    (a column's chirp-z transform is indivisible; tiling the OUTPUT Doppler bins instead would repeat the
    whole transform on every rank) and the tiles are gathered to ``dst`` and assembled into the Map.
    Returns the [nDop, nDel] complex64 map on ``dst``, None elsewhere.
    ``amb`` needs ``geometry``, ``range_device`` and ``doppler_device`` (blah2_b200.process.Ambiguity).
    """
    g = amb.geometry
    n_dop, n_del, n_corr = g.n_doppler_bins, g.n_delay_bins, g.n_corr
    b0, nb = block_range(n_dop, rank, world)
    assert d_x_local.numel() == nb * n_corr and d_y_local.numel() == nb * n_corr, "local IQ must hold exactly the rank's batches"
    dev = d_x_local.device
    # The torch operations around the two kernels (copies, collectives, transposes) run on torch's CURRENT stream;
    # the kernels must be ordered with them, so without an explicit stream they go onto that one -- never onto the
    # handle's private non-blocking stream (ADVICE r1).  An explicit stream must be current while this runs.
    if stream is None and dev.type == "cuda":
        stream = torch.cuda.current_stream(dev)
    s_ptr = stream.cuda_stream if stream is not None and hasattr(stream, "cuda_stream") else stream
    R_local = torch.empty((nb, n_del), dtype=torch.complex64, device=dev)
    amb.range_device(d_x_local, d_y_local, b0, nb, R_local, s_ptr)
    if world > 1:
        counts = [block_range(n_dop, r, world)[1] for r in range(world)]
        R_full = _all_gather_rows(R_local, counts, world)
    else:
        R_full = R_local
    c0, nc = block_range(n_del, rank, world)
    tile = torch.empty((n_dop, nc), dtype=torch.complex64, device=dev)
    amb.doppler_device(R_full.contiguous(), c0, nc, tile, s_ptr)
    if world == 1:
        return tile
    ccounts = [block_range(n_del, r, world)[1] for r in range(world)]
    k_max = max(ccounts)
    buf = torch.zeros((k_max, n_dop), dtype=torch.complex64, device=dev)
    buf[:nc] = tile.transpose(0, 1)
    flat = torch.view_as_real(buf).contiguous()
    gathered = [torch.empty_like(flat) for _ in range(world)] if rank == dst else None
    dist.gather(flat, gathered, dst=dst)
    if rank != dst:
        return None
    cols = torch.cat([torch.view_as_complex(gathered[r])[: ccounts[r]] for r in range(world)], dim=0)  # [nDel, nDop]
    return cols.transpose(0, 1).contiguous()


# ------------------------------------------------------------------------------------------
# Same interface as Comm on top of torch.distributed (gloo): CPU tests of the orchestration below
# ------------------------------------------------------------------------------------------
class TorchComm:
    """Synchronous stand-in for Comm (tests/test_shard_cpu.py, world_size-2 gloo on CPU tensors)."""

    def __init__(self, rank: int, world: int):
        self.rank, self.world = rank, world

    @staticmethod
    def _bytes(t):
        return torch.view_as_real(t).reshape(-1) if t.is_complex() else t.reshape(-1)

    def gather_async(self, send, recv, dst=0, after=None):
        got = [torch.empty_like(self._bytes(send)) for _ in range(self.world)] if self.rank == dst else None
        dist.gather(self._bytes(send).contiguous(), got, dst=dst)
        if self.rank == dst:
            for r in range(self.world):
                self._bytes(recv[r]).copy_(got[r])

    def gatherv_async(self, send, recv, sizes, offsets, dst=0, after=None):
        es = send.element_size()
        parts = None
        if self.rank == dst:
            parts = [torch.empty(int(sizes[r]) // es, dtype=send.dtype) for r in range(self.world)]
        # gloo's gather wants equal sizes: pad to the largest block
        k = max(int(v) for v in sizes) // es
        buf = torch.zeros(k, dtype=send.dtype)
        buf[: send.numel()] = send.reshape(-1)
        got = [torch.empty_like(self._bytes(buf)) for _ in range(self.world)] if self.rank == dst else None
        dist.gather(self._bytes(buf).contiguous(), got, dst=dst)
        if self.rank == dst:
            flat = recv.reshape(-1)
            for r in range(self.world):
                n_r = int(sizes[r]) // es
                blk = got[r]
                blk = torch.view_as_complex(blk.reshape(-1, 2)) if send.is_complex() else blk
                flat[int(offsets[r]) // es: int(offsets[r]) // es + n_r] = blk[:n_r]

    def allgatherv_async(self, send, recv, sizes, offsets, after=None):
        es = send.element_size()
        k = max(int(v) for v in sizes) // es
        buf = torch.zeros(k, dtype=send.dtype)
        buf[: send.numel()] = send.reshape(-1)
        got = [torch.empty_like(self._bytes(buf)) for _ in range(self.world)]
        dist.all_gather(got, self._bytes(buf).contiguous())
        flat = recv.reshape(-1)
        for r in range(self.world):
            n_r = int(sizes[r]) // es
            blk = torch.view_as_complex(got[r].reshape(-1, 2)) if send.is_complex() else got[r]
            flat[int(offsets[r]) // es: int(offsets[r]) // es + n_r] = blk[:n_r]

    def allreduce_f64_async(self, buf, after=None):
        t = self._bytes(buf)
        dist.all_reduce(t)

    def sendrecv_async(self, send, send_peer, recv, recv_peer, after=None):
        ops = []
        if send is not None and send_peer >= 0 and send.numel():
            if send_peer == self.rank and recv_peer == self.rank:
                recv.copy_(send)
                return
            ops.append(dist.isend(self._bytes(send).contiguous(), send_peer))
        tmp = None
        if recv is not None and recv_peer >= 0 and recv.numel():
            tmp = torch.empty_like(self._bytes(recv))
            ops.append(dist.irecv(tmp, recv_peer))
        for o in ops:
            o.wait()
        if tmp is not None:
            self._bytes(recv).copy_(tmp) if recv.is_contiguous() else recv.copy_(torch.view_as_complex(tmp.reshape(-1, 2)).reshape(recv.shape))

    def join(self, stream):
        pass

    def sync(self):
        pass


class SingleCpiPlan:
    """ONE large CPI split over the ranks (BASELINE config 5), clutter filter included (SURVEY.md s8e rows 2-3).

    Rank r owns a contiguous block of batches -- samples [s0, s0 + ns) of the CPI, the last rank also the
    N - nDop nCorr samples the Ambiguity stage leaves over (the filter runs over all N).  Per CPI:
      1. [filter] halo exchange with the two neighbours (b200dd_comm_sendrecv_async), per-chunk correlations,
         all-reduce of the 2 nBins sums, replicated solve, per-chunk filter          (WienerHopf.cpp:58-163);
      2. range correlation of the rank's batches into its rows of the range matrix    (Ambiguity.cpp:106-149);
      3. all-gather of the range matrix (nDop x nDel complex64, <= 17 MB) -- the one exchange the CAF needs:
         the Doppler transform runs ALONG the batch axis;
      4. Doppler transform of the rank's tile of delay columns                         (Ambiguity.cpp:152-169);
      5. gather of the tiles to rank `dst`, placed into the row-major map.
    All buffers are allocated here, once; `run` only enqueues kernels and exchanges (`comm` is a blah2_b200.shard.Comm
    on GPUs, a TorchComm in the CPU tests; `amb` / `whc_factory` are the process-layer classes or CPU stand-ins).

    Every product of the CPI on `dst`: ``spectrum`` (every rank) is a SpectrumAnalyser(n_samples, bandwidth); each
    rank folds its samples [s0, s0 + ns) below nfft into one part of the spectrum, and the parts are gathered to
    `dst` in rank order.  ``pipeline`` (rank `dst` only) is the importing Pipeline, created with the full parameters:
    `run` stamps its stage boundaries and ends with pipeline.submit_map of the placed map, the chunk's clutter-filter
    verdict and the parts; the caller then fetches on `dst` as from any pipeline.  The plan reuses its map and part
    buffers, so a run must follow the fetch of the previous CPI."""

    def __init__(self, comm, amb, n_samples: int, device, clutter=None, whc_factory=None, dst: int = 0,
                 spectrum=None, pipeline=None):
        self.comm, self.amb, self.dst = comm, amb, dst
        self.spectrum, self.pipeline = spectrum, pipeline
        rank, world = comm.rank, comm.world
        g = amb.geometry
        self.n_dop, self.n_del, self.n_corr = g.n_doppler_bins, g.n_delay_bins, g.n_corr
        n_used = self.n_dop * self.n_corr
        self.b0, self.nb = block_range(self.n_dop, rank, world)
        self.s0 = self.b0 * self.n_corr
        self.ns = self.nb * self.n_corr + (n_samples - n_used if rank == world - 1 else 0)
        c64 = torch.complex64
        self.R_full = torch.zeros((self.n_dop, self.n_del), dtype=c64, device=device)
        self.R_local = self.R_full[self.b0:self.b0 + self.nb]          # the rank's rows, in place
        self.row_sizes = [block_range(self.n_dop, r, world)[1] * self.n_del * 8 for r in range(world)]
        self.row_offsets = [block_range(self.n_dop, r, world)[0] * self.n_del * 8 for r in range(world)]
        self.c0, self.nc = block_range(self.n_del, rank, world)
        self.tile = torch.zeros((self.n_dop, self.nc), dtype=c64, device=device)
        cols = [block_range(self.n_del, r, world) for r in range(world)]
        self.tile_sizes = [self.n_dop * c[1] * 8 for c in cols]
        self.tile_offsets = [self.n_dop * c[0] * 8 for c in cols]
        self.cols = cols
        self.tiles_all = torch.zeros(self.n_dop * self.n_del, dtype=c64, device=device) if rank == dst else None
        self.map = torch.zeros((self.n_dop, self.n_del), dtype=c64, device=device) if rank == dst else None
        # clutter filter on the rank's chunk
        self.whc = None
        if clutter is not None:
            self.whc = whc_factory(clutter[0], clutter[1], n_samples, self.s0, self.ns)
            xl, xr, yr = self.whc.halos()
            self.xl, self.xr, self.yr = xl, xr, yr
            self.x_loc = torch.zeros(xl + self.ns + xr, dtype=c64, device=device)
            self.y_loc = torch.zeros(self.ns + yr, dtype=c64, device=device)
            self.ab = torch.zeros(2 * self.whc.nBins, dtype=torch.complex128, device=device)
            self.y_f = torch.zeros(self.ns, dtype=c64, device=device)
            self.x_own = self.x_loc[xl:xl + self.ns]     # the caller writes its samples HERE (no staging copy)
            self.y_own = self.y_loc[:self.ns]
        else:
            self.x_own = torch.zeros(self.ns, dtype=c64, device=device)
            self.y_own = torch.zeros(self.ns, dtype=c64, device=device)
        if spectrum is not None:
            # the rank's samples below nfft (none when the slice starts past it)
            self.n_fold = max(0, min(self.ns, spectrum.nfft - self.s0))
            self.part = torch.zeros(spectrum.nSpectrum, dtype=torch.complex128, device=device)
            self.parts = torch.zeros((world, spectrum.nSpectrum), dtype=torch.complex128, device=device) \
                if rank == dst else None

    def run(self, stream=None, marks=None):
        """Process the CPI whose samples are in x_own / y_own.  Returns the [nDop, nDel] map on `dst`, None elsewhere
        (valid once `stream` has drained).  `marks` (a list) receives (label, event) pairs recorded on `stream`
        after each stage, for the per-stage timing of tools/bench_cfg5.py."""
        comm, rank, world = self.comm, self.comm.rank, self.comm.world
        sp = stream.cuda_stream if hasattr(stream, "cuda_stream") else stream

        def mark(label):
            if marks is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record(stream)
                marks.append((label, e))
        mark("start")
        pipe = self.pipeline if rank == self.dst else None
        if pipe is not None:
            pipe.stamp(STAMP_CHAIN, sp)
        if self.spectrum is not None:
            self.spectrum.fold_slice_device(self.x_own[:self.n_fold], self.s0, self.part, sp)
            comm.gather_async(self.part, self.parts, self.dst, after=stream)
            mark("spectrum")
        if pipe is not None:
            pipe.stamp(STAMP_SPECTRUM, sp)
        x, y = self.x_own, self.y_own
        if self.whc is not None:
            nxt, prv = (rank + 1) % world, (rank - 1) % world
            # right halos (circular: the correlations are circular over N): my first samples go to the previous rank
            comm.sendrecv_async(self.x_own[:self.xr], prv, self.x_loc[self.xl + self.ns:], nxt, after=stream)
            comm.sendrecv_async(self.y_own[:self.yr], prv, self.y_loc[self.ns:], nxt, after=None)
            # left halo = filter history (not circular: zero before sample 0): my last samples go to the next rank
            if self.xl:
                comm.sendrecv_async(self.x_own[self.ns - self.xl:], nxt if rank + 1 < world else -1, self.x_loc[:self.xl],
                                    prv if rank > 0 else -1, after=None)
            comm.join(stream)
            mark("halo")
            self.whc.corr_device(self.x_loc, self.y_loc, self.ab, sp)
            mark("wh_corr")
            comm.allreduce_f64_async(self.ab, after=stream)
            comm.join(stream)
            mark("allreduce")
            self.whc.filter_device(self.ab, self.x_loc, self.y_loc, self.y_f, sp)
            mark("wh_solve_filter")
            y = self.y_f
        if pipe is not None:
            pipe.stamp(STAMP_CLUTTER, sp)
        n_own = self.nb * self.n_corr
        self.amb.range_device(x[:n_own], y[:n_own], self.b0, self.nb, self.R_local, sp)
        mark("range")
        comm.allgatherv_async(self.R_local, self.R_full, self.row_sizes, self.row_offsets, after=stream)
        comm.join(stream)
        mark("allgather_R")
        self.amb.doppler_device(self.R_full, self.c0, self.nc, self.tile, sp)
        mark("doppler")
        comm.gatherv_async(self.tile, self.tiles_all, self.tile_sizes, self.tile_offsets, self.dst, after=stream)
        if rank != self.dst:
            return None
        comm.join(stream)
        mark("gather_tiles")
        if hasattr(self.amb, "place_tiles"):       # tiles -> columns of the row-major map: one kernel
            self.amb.place_tiles(self.tiles_all, world, self.map, sp)
        else:
            for r, (c0, nc) in enumerate(self.cols):
                off = self.tile_offsets[r] // 8
                self.amb.place_tile(self.tiles_all[off:off + self.n_dop * nc], c0, nc, self.map, sp)
        mark("place_tiles")
        if pipe is not None:
            pipe.submit_map(self.map, self.whc.device_status() if self.whc is not None else None,
                            self.parts if self.spectrum is not None else None, sp)
            mark("submit_map")
        return self.map
