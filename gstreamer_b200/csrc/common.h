// gstreamer_b200/csrc/common.h — shared helpers of libb200dsp (product code).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#include "../../include/b200dsp.h"

namespace b200 {

// records the failing call for b200_last_cuda_error(); returns B200_ERR_CUDA
int cuda_fail (cudaError_t e, const char *what, const char *file, int line);

#define B200_CUDA_TRY(expr)                                              \
  do {                                                                   \
    cudaError_t e__ = (expr);                                            \
    if (e__ != cudaSuccess)                                              \
      return ::b200::cuda_fail (e__, #expr, __FILE__, __LINE__);         \
  } while (0)

// RAII device selection: the C-ABI lets each handle live on its own device
// (one pipeline per GPU), so every entry point pins the device for its duration.
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard (int dev) {
    if (cudaGetDevice (&prev) != cudaSuccess) { prev = -1; }
    if (dev != prev && cudaSetDevice (dev) != cudaSuccess) ok = false;
  }
  ~DeviceGuard () { if (prev >= 0) cudaSetDevice (prev); }
};

// Opt a kernel in to the device's full dynamic shared memory.  The attribute is per FUNCTION (and per device), not per
// handle: plans of different footprints share the kernels, so the limit is always raised to the device's opt-in maximum
// (227 KB on sm_90) and never to one plan's own size — a later, smaller handle must not lower it under an earlier one.
// The limit itself costs nothing; occupancy follows the bytes each launch actually asks for.
template <typename F>
int allow_max_dyn_smem (F fn)
{
  int dev = 0, optin = 0;
  B200_CUDA_TRY (cudaGetDevice (&dev));
  B200_CUDA_TRY (cudaDeviceGetAttribute (&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  cudaFuncAttributes fa;
  B200_CUDA_TRY (cudaFuncGetAttributes (&fa, fn));               // static shared memory counts against the same limit
  B200_CUDA_TRY (cudaFuncSetAttribute (fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int) fa.sharedSizeBytes));
  return B200_OK;
}

// number of SMs of a device (cached)
int sm_count (int device);

template <typename T>
int upload (T **dptr, const T *host, size_t n)
{
  if (n == 0) { *dptr = nullptr; return B200_OK; }
  B200_CUDA_TRY (cudaMalloc ((void **) dptr, n * sizeof (T)));
  B200_CUDA_TRY (cudaMemcpy (*dptr, host, n * sizeof (T), cudaMemcpyHostToDevice));
  return B200_OK;
}

}  // namespace b200
