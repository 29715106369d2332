// comm.cu -- the path's few inter-GPU exchanges, issued from C on a dedicated communication stream.
//
// The reference has no distributed code (SURVEY.md s2b); the sharding is ours (SURVEY.md s8e):
//   * a stream of independent CPIs round-robin over the GPUs: the ONLY communication is the gather of finished
//     maps to rank 0 (b200dd_comm_gather_async), overlapped with the next CPI's kernels;
//   * one large CPI split over the GPUs: all-gather of the range matrix between the two CAF stages, gather of the
//     delay-column tiles, and for the clutter filter an all-reduce of the 2 nBins partial correlations plus an
//     nBins-sample halo from the left neighbour (b200dd_comm_allgatherv_async, _allreduce_f64_async,
//     _sendrecv_async).
// One process per GPU; the communicator is NCCL over NVLink / NVSwitch.  NCCL is resolved at run time with
// dlopen("libnccl.so.2") -- the single-GPU library has no link-time dependency on it, and inside a process that
// already loaded a NCCL (PyTorch's bundled one) the same copy is reused.  Every call enqueues on the
// communicator's own non-blocking stream after an event recorded on the caller's compute stream (`after`), and
// returns; b200dd_comm_join makes a compute stream wait for what has been enqueued so far.
#include "common.cuh"

#include <dlfcn.h>

#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <vector>

using namespace b2;

namespace {

// Minimal NCCL ABI (nccl.h of NCCL 2.7 .. 2.28: these declarations have not changed)
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclSuccess = 0 };
enum { ncclUint8 = 1, ncclFloat64 = 8 };
enum { ncclSum = 0 };

struct NcclApi {
  void *lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Send)(const void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  std::string error;
};

NcclApi &nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {
      api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.lib) break;
    }
    if (!api.lib) {
      api.error = std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : "");
      return;
    }
    auto sym = [&](const char *n) {
      void *p = dlsym(api.lib, n);
      if (!p && api.error.empty()) api.error = std::string("NCCL symbol missing: ") + n;
      return p;
    };
    api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
    api.Send = (decltype(api.Send))sym("ncclSend");
    api.Recv = (decltype(api.Recv))sym("ncclRecv");
    api.Broadcast = (decltype(api.Broadcast))sym("ncclBroadcast");
    api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
    api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
    api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
    api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
  });
  return api;
}

int nccl_fail(ncclResult_t r, const char *what) {
  NcclApi &a = nccl_api();
  set_last_error(std::string(what) + " failed: " + (a.GetErrorString ? a.GetErrorString(r) : "NCCL error"));
  return B200DD_ERR_CUDA;
}

#define B2_NCCL(expr)                                      \
  do {                                                     \
    ncclResult_t _r = (expr);                              \
    if (_r != ncclSuccess) return nccl_fail(_r, #expr);    \
  } while (0)

}  // namespace

struct b200dd_comm {
  int rank = 0, world = 1, device = 0;
  Stream stream;
  Event ev_in, ev_out;
  ncclComm_t comm = nullptr;
};

namespace {

// order the communication stream after everything enqueued so far on the caller's compute stream
int comm_after(b200dd_comm *c, void *after) {
  if (after) {
    B2_CUDA(cudaEventRecord(c->ev_in, (cudaStream_t)after));
    B2_CUDA(cudaStreamWaitEvent(c->stream, c->ev_in, 0));
  }
  return B200DD_OK;
}

}  // namespace

extern "C" {

int b200dd_comm_get_unique_id(uint8_t *id128) {
  if (!id128) return arg_fail("b200dd_comm_get_unique_id: null argument");
  NcclApi &a = nccl_api();
  if (!a.error.empty()) { set_last_error(a.error); return B200DD_ERR_CUDA; }
  ncclUniqueId id;
  B2_NCCL(a.GetUniqueId(&id));
  memcpy(id128, id.internal, 128);
  return B200DD_OK;
}

int b200dd_comm_create(int32_t rank, int32_t world, const uint8_t *id128, int32_t device, b200dd_comm **out) {
  if (!out || !id128) return arg_fail("b200dd_comm_create: null argument");
  *out = nullptr;
  if (world < 1 || rank < 0 || rank >= world) return arg_fail("b200dd_comm_create: bad rank / world");
  NcclApi &a = nccl_api();
  if (!a.error.empty()) { set_last_error(a.error); return B200DD_ERR_CUDA; }
  Owned<b200dd_comm> c(new (std::nothrow) b200dd_comm(), b200dd_comm_destroy);
  if (!c) return arg_fail("b200dd_comm_create: out of host memory");
  c->rank = rank;
  c->world = world;
  if (int rc = resolve_device(device, &c->device)) return rc;
  DeviceGuard guard(c->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  B2_CUDA(c->stream.create());
  B2_CUDA(c->ev_in.create(cudaEventDisableTiming));
  B2_CUDA(c->ev_out.create(cudaEventDisableTiming));
  ncclUniqueId id;
  memcpy(id.internal, id128, 128);
  // The exchanges of this path are small (a map, a range matrix, a halo) and run BESIDE kernels that need whole SMs
  // (255 registers x 256 threads): every channel is a resident CTA that spins while it waits for its peer.  Two
  // point-to-point channels carry the ~1 MB messages at NVLink speed; the caller's own NCCL_* settings win.
  setenv("NCCL_MAX_P2P_NCHANNELS", "2", 0);
  setenv("NCCL_MIN_P2P_NCHANNELS", "1", 0);
  B2_NCCL(a.CommInitRank(&c->comm, world, id, rank));
  *out = c.release();
  return B200DD_OK;
}

void b200dd_comm_destroy(b200dd_comm *c) {
  if (!c) return;
  DeviceGuard guard(c->device);  // held while the members go
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->comm) nccl_api().CommDestroy(c->comm);
  delete c;
}

int32_t b200dd_comm_rank(const b200dd_comm *c) { return c ? c->rank : -1; }
int32_t b200dd_comm_world(const b200dd_comm *c) { return c ? c->world : 0; }
void *b200dd_comm_stream(b200dd_comm *c) { return c ? (void *)c->stream : nullptr; }

int b200dd_comm_gather_async(b200dd_comm *c, const void *d_send, void *d_recv, size_t bytes, int32_t dst, void *after) {
  if (!c || !d_send) return arg_fail("b200dd_comm_gather_async: null argument");
  if (dst < 0 || dst >= c->world) return arg_fail("b200dd_comm_gather_async: bad destination rank");
  if (c->rank == dst && !d_recv) return arg_fail("b200dd_comm_gather_async: the destination rank needs a receive buffer");
  DeviceGuard guard(c->device);
  int rc = comm_after(c, after);
  if (rc != B200DD_OK) return rc;
  NcclApi &a = nccl_api();
  if (c->rank == dst) {
    B2_CUDA(cudaMemcpyAsync((char *)d_recv + (size_t)dst * bytes, d_send, bytes, cudaMemcpyDeviceToDevice, c->stream));
    if (c->world > 1) {
      B2_NCCL(a.GroupStart());
      for (int r = 0; r < c->world; r++)
        if (r != dst) B2_NCCL(a.Recv((char *)d_recv + (size_t)r * bytes, bytes, ncclUint8, r, c->comm, c->stream));
      B2_NCCL(a.GroupEnd());
    }
  } else {
    B2_NCCL(a.Send(d_send, bytes, ncclUint8, dst, c->comm, c->stream));
  }
  return B200DD_OK;
}

int b200dd_comm_gatherv_async(b200dd_comm *c, const void *d_send, size_t send_bytes, void *d_recv, const size_t *bytes,
                              const size_t *offsets, int32_t dst, void *after) {
  if (!c || !d_send) return arg_fail("b200dd_comm_gatherv_async: null argument");
  if (dst < 0 || dst >= c->world) return arg_fail("b200dd_comm_gatherv_async: bad destination rank");
  if (c->rank == dst && (!d_recv || !bytes || !offsets)) return arg_fail("b200dd_comm_gatherv_async: the destination rank needs receive buffer, sizes and offsets");
  DeviceGuard guard(c->device);
  int rc = comm_after(c, after);
  if (rc != B200DD_OK) return rc;
  NcclApi &a = nccl_api();
  if (c->rank == dst) {
    if (bytes[dst] != send_bytes) return arg_fail("b200dd_comm_gatherv_async: own block size mismatch");
    if (send_bytes) B2_CUDA(cudaMemcpyAsync((char *)d_recv + offsets[dst], d_send, send_bytes, cudaMemcpyDeviceToDevice, c->stream));
    if (c->world > 1) {
      B2_NCCL(a.GroupStart());
      for (int r = 0; r < c->world; r++)
        if (r != dst && bytes[r]) B2_NCCL(a.Recv((char *)d_recv + offsets[r], bytes[r], ncclUint8, r, c->comm, c->stream));
      B2_NCCL(a.GroupEnd());
    }
  } else if (send_bytes) {
    B2_NCCL(a.Send(d_send, send_bytes, ncclUint8, dst, c->comm, c->stream));
  }
  return B200DD_OK;
}

int b200dd_comm_allgatherv_async(b200dd_comm *c, const void *d_send, void *d_recv, const size_t *bytes,
                                 const size_t *offsets, void *after) {
  if (!c || !d_send || !d_recv || !bytes || !offsets) return arg_fail("b200dd_comm_allgatherv_async: null argument");
  DeviceGuard guard(c->device);
  int rc = comm_after(c, after);
  if (rc != B200DD_OK) return rc;
  NcclApi &a = nccl_api();
  char *own = (char *)d_recv + offsets[c->rank];
  if ((const void *)own != d_send && bytes[c->rank])
    B2_CUDA(cudaMemcpyAsync(own, d_send, bytes[c->rank], cudaMemcpyDeviceToDevice, c->stream));
  if (c->world > 1) {
    // every rank sends its block to every other rank and receives theirs: one group = one launch, each pair on its
    // own NVLink path through the switch
    B2_NCCL(a.GroupStart());
    for (int r = 0; r < c->world; r++) {
      if (r == c->rank) continue;
      if (bytes[c->rank]) B2_NCCL(a.Send(own, bytes[c->rank], ncclUint8, r, c->comm, c->stream));
      if (bytes[r]) B2_NCCL(a.Recv((char *)d_recv + offsets[r], bytes[r], ncclUint8, r, c->comm, c->stream));
    }
    B2_NCCL(a.GroupEnd());
  }
  return B200DD_OK;
}

int b200dd_comm_allreduce_f64_async(b200dd_comm *c, void *d_buf, size_t count, void *after) {
  if (!c || !d_buf) return arg_fail("b200dd_comm_allreduce_f64_async: null argument");
  DeviceGuard guard(c->device);
  int rc = comm_after(c, after);
  if (rc != B200DD_OK) return rc;
  if (c->world > 1) B2_NCCL(nccl_api().AllReduce(d_buf, d_buf, count, ncclFloat64, ncclSum, c->comm, c->stream));
  return B200DD_OK;
}

int b200dd_comm_sendrecv_async(b200dd_comm *c, const void *d_send, size_t send_bytes, int32_t send_peer, void *d_recv,
                               size_t recv_bytes, int32_t recv_peer, void *after) {
  if (!c) return arg_fail("b200dd_comm_sendrecv_async: null handle");
  const bool do_send = send_peer >= 0 && send_bytes > 0, do_recv = recv_peer >= 0 && recv_bytes > 0;
  if ((do_send && (!d_send || send_peer >= c->world)) || (do_recv && (!d_recv || recv_peer >= c->world)))
    return arg_fail("b200dd_comm_sendrecv_async: bad peer or null buffer");
  DeviceGuard guard(c->device);
  int rc = comm_after(c, after);
  if (rc != B200DD_OK) return rc;
  NcclApi &a = nccl_api();
  if (do_send && do_recv && send_peer == c->rank && recv_peer == c->rank) {  // talking to oneself (world == 1 rings)
    if (send_bytes != recv_bytes) return arg_fail("b200dd_comm_sendrecv_async: self exchange with different sizes");
    B2_CUDA(cudaMemcpyAsync(d_recv, d_send, send_bytes, cudaMemcpyDeviceToDevice, c->stream));
    return B200DD_OK;
  }
  B2_NCCL(a.GroupStart());
  ncclResult_t r1 = ncclSuccess, r2 = ncclSuccess;
  if (do_send) r1 = a.Send(d_send, send_bytes, ncclUint8, send_peer, c->comm, c->stream);
  if (do_recv) r2 = a.Recv(d_recv, recv_bytes, ncclUint8, recv_peer, c->comm, c->stream);
  B2_NCCL(a.GroupEnd());
  if (r1 != ncclSuccess) return nccl_fail(r1, "ncclSend");
  if (r2 != ncclSuccess) return nccl_fail(r2, "ncclRecv");
  return B200DD_OK;
}

int b200dd_comm_wait_stream(b200dd_comm *c, void *stream) {
  if (!c || !stream) return arg_fail("b200dd_comm_wait_stream: null argument");
  DeviceGuard guard(c->device);
  return comm_after(c, stream);
}

int b200dd_comm_join(b200dd_comm *c, void *stream) {
  if (!c || !stream) return arg_fail("b200dd_comm_join: null argument");
  DeviceGuard guard(c->device);
  B2_CUDA(cudaEventRecord(c->ev_out, c->stream));
  B2_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, c->ev_out, 0));
  return B200DD_OK;
}

int b200dd_comm_sync(b200dd_comm *c) {
  if (!c) return arg_fail("b200dd_comm_sync: null handle");
  DeviceGuard guard(c->device);
  B2_CUDA(cudaStreamSynchronize(c->stream));
  return B200DD_OK;
}

}  // extern "C"
