// hostutil.cu -- host-side placement helper: the end-to-end path is PCIe-bound (64 MB per CPI), and a submitting
// thread / pinned staging buffer on the far NUMA node costs a large share of the copy bandwidth.  b200dd_bind_host_to_device pins the calling thread to the CPUs the kernel lists as local to
// the GPU's PCIe root (sysfs local_cpulist); pinned memory allocated afterwards lands on that node (first touch).
#include "common.cuh"

#include <sched.h>

#include <cctype>
#include <cstdlib>
#include <cstring>
#include <string>

using namespace b2;

extern "C" int b200dd_bind_host_to_device(int32_t device, char *cpulist_out, int32_t cap) {
  int dev;
  if (int rc = resolve_device(device, &dev)) return rc;
  char bus[32] = {0};
  B2_CUDA(cudaDeviceGetPCIBusId(bus, sizeof(bus), dev));
  for (char *p = bus; *p; p++) *p = (char)tolower(*p);
  const std::string path = std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist";
  FILE *f = fopen(path.c_str(), "r");
  if (!f) { set_last_error("b200dd_bind_host_to_device: cannot read " + path); return B200DD_ERR_ARG; }
  char line[4096] = {0};
  const bool got = fgets(line, sizeof(line), f) != nullptr;
  fclose(f);
  if (!got) { set_last_error("b200dd_bind_host_to_device: empty " + path); return B200DD_ERR_ARG; }
  line[strcspn(line, "\r\n")] = 0;
  if (cpulist_out && cap > 0) {
    strncpy(cpulist_out, line, (size_t)cap - 1);
    cpulist_out[cap - 1] = 0;
  }
  cpu_set_t want, have;
  CPU_ZERO(&want);
  if (sched_getaffinity(0, sizeof(have), &have) != 0) CPU_ZERO(&have);
  int n = 0;
  for (char *tok = strtok(line, ","); tok; tok = strtok(nullptr, ",")) {  // "0-31,64-95"
    int a = 0, b = 0;
    if (sscanf(tok, "%d-%d", &a, &b) == 2) {
    } else if (sscanf(tok, "%d", &a) == 1) {
      b = a;
    } else {
      continue;
    }
    for (int c = a; c <= b && c < CPU_SETSIZE; c++)
      if (CPU_ISSET(c, &have)) { CPU_SET(c, &want); n++; }  // never widen what the caller (a container cgroup) allows
  }
  if (n == 0) return B200DD_OK;  // nothing local is allowed: leave the affinity alone
  if (sched_setaffinity(0, sizeof(want), &want) != 0) { set_last_error("b200dd_bind_host_to_device: sched_setaffinity failed"); return B200DD_ERR_ARG; }
  return B200DD_OK;
}

// Pinned (page-locked) host memory for the drop-in classes' staging buffers: a pageable std::vector crosses PCIe at a
// third of the pinned rate.  Plain malloc/free semantics; NULL on failure.
extern "C" void *b200dd_host_alloc(size_t bytes) {
  void *p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
extern "C" void b200dd_host_free(void *p) {
  if (p) cudaFreeHost(p);
}
