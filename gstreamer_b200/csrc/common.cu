// gstreamer_b200/csrc/common.cu — status strings, device helpers, pinned host memory.
#include "common.h"

#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <unistd.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <map>
#include <mutex>

namespace b200 {

static thread_local char g_last_cuda[512] = "";

int cuda_fail (cudaError_t e, const char *what, const char *file, int line)
{
  snprintf (g_last_cuda, sizeof (g_last_cuda), "%s:%d: %s -> %s (%s)", file, line, what,
      cudaGetErrorName (e), cudaGetErrorString (e));
  // clear the sticky-less error state so later calls report their own failures
  cudaGetLastError ();
  if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver)
    return B200_ERR_NO_DEVICE;
  if (e == cudaErrorMemoryAllocation)
    return B200_ERR_NOMEM;
  return B200_ERR_CUDA;
}

int sm_count (int device)
{
  static int cache[64];
  if (device < 0 || device >= 64) return 132;
  if (cache[device] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute (&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0)
      n = 132;                                      // H100 SXM
    cache[device] = n;
  }
  return cache[device];
}

}  // namespace b200

extern "C" {

const char *b200_strerror (int status)
{
  switch (status) {
    case B200_OK: return "ok";
    case B200_ERR_INVALID_ARG: return "invalid argument";
    case B200_ERR_UNSUPPORTED: return "unsupported format or mode";
    case B200_ERR_NO_DEVICE: return "no CUDA device (libb200dsp has no CPU fallback)";
    case B200_ERR_CUDA: return "CUDA call failed";
    case B200_ERR_NOMEM: return "out of memory";
    case B200_ERR_STATE: return "invalid handle state";
    default: return "unknown status";
  }
}

const char *b200_last_cuda_error (void) { return b200::g_last_cuda; }

int b200_version (void) { return B200DSP_VERSION_MAJOR * 100 + B200DSP_VERSION_MINOR; }

int b200_device_count (void)
{
  int n = 0;
  cudaError_t e = cudaGetDeviceCount (&n);
  if (e != cudaSuccess)
    return b200::cuda_fail (e, "cudaGetDeviceCount", __FILE__, __LINE__);
  return n;
}

// NUMA node of a device's PCIe root, from sysfs (-1: unknown / single node)
int b200_device_numa_node (int device)
{
  char bus[32] = "", path[128];
  if (device < 0 || cudaDeviceGetPCIBusId (bus, sizeof (bus), device) != cudaSuccess) { cudaGetLastError (); return -1; }
  for (char *c = bus; *c; c++) if (*c >= 'A' && *c <= 'Z') *c += 'a' - 'A';      // sysfs names are lower case
  snprintf (path, sizeof (path), "/sys/bus/pci/devices/%s/numa_node", bus);
  FILE *f = fopen (path, "r");
  if (!f) return -1;
  int node = -1;
  if (fscanf (f, "%d", &node) != 1) node = -1;
  fclose (f);
  return node;
}

namespace {
std::mutex g_reg_lock;
std::map<void *, size_t> g_registered;      // mmap'ed + cudaHostRegister'ed blocks of b200_host_alloc_near
}

// Staging memory on the NUMA node the device hangs off: with one pipeline per GPU on a two-socket host, page-locked
// buffers that happen to sit on the other socket push every H2D / D2H byte across the socket interconnect.
// Pages are bound with mbind(MPOL_BIND) BEFORE they are touched,
// then locked and mapped with cudaHostRegister - the placement does not depend on which core the caller runs on.
int b200_host_alloc_near (int device, size_t size, void **ptr)
{
  if (!ptr || size == 0) return B200_ERR_INVALID_ARG;
  *ptr = nullptr;
  const int node = b200_device_numa_node (device);
  if (node < 0 || node >= 1024) {                                  // no topology information: plain pinned memory
    B200_CUDA_TRY (cudaHostAlloc (ptr, size, cudaHostAllocPortable));
    return B200_OK;
  }
  // 2 MB granules + MADV_HUGEPAGE: transparent huge pages where the host allows them (fewer, larger DMA mappings)
  const size_t page = (size_t) 2 << 20;
  const size_t bytes = (size + page - 1) / page * page;
  void *p = mmap (nullptr, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  if (p == MAP_FAILED) return B200_ERR_NOMEM;
  (void) madvise (p, bytes, MADV_HUGEPAGE);
  unsigned long mask[16] = {0};
  mask[node / (8 * sizeof (unsigned long))] = 1ul << (node % (8 * sizeof (unsigned long)));
  // MPOL_BIND = 2; a kernel without NUMA support fails here and the pages simply follow the default policy
  (void) syscall (SYS_mbind, p, bytes, 2, mask, (unsigned long) (8 * sizeof (mask)), 0u);
  memset (p, 0, bytes);                                            // first touch: pages now exist on `node`
  cudaError_t e = cudaHostRegister (p, bytes, cudaHostRegisterPortable);
  if (e != cudaSuccess) {
    munmap (p, bytes);
    return b200::cuda_fail (e, "cudaHostRegister", __FILE__, __LINE__);
  }
  {
    std::lock_guard<std::mutex> lk (g_reg_lock);
    g_registered[p] = bytes;
  }
  *ptr = p;
  return B200_OK;
}

int b200_host_alloc (size_t size, void **ptr)
{
  int dev = -1;
  if (cudaGetDevice (&dev) != cudaSuccess) { cudaGetLastError (); dev = -1; }
  return b200_host_alloc_near (dev, size, ptr);
}

int b200_host_free (void *ptr)
{
  if (!ptr) return B200_OK;
  size_t bytes = 0;
  {
    std::lock_guard<std::mutex> lk (g_reg_lock);
    auto it = g_registered.find (ptr);
    if (it != g_registered.end ()) { bytes = it->second; g_registered.erase (it); }
  }
  if (bytes) {
    cudaError_t e = cudaHostUnregister (ptr);
    munmap (ptr, bytes);
    if (e != cudaSuccess) return b200::cuda_fail (e, "cudaHostUnregister", __FILE__, __LINE__);
    return B200_OK;
  }
  B200_CUDA_TRY (cudaFreeHost (ptr));
  return B200_OK;
}

}  // extern "C"
