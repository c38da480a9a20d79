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

#define B200_CUDA_RET(expr)                                              \
  do {                                                                   \
    cudaError_t e__ = (expr);                                            \
    if (e__ != cudaSuccess) return e__;                                  \
  } while (0)

// The staging ring of the system-memory entry points (DESIGN.md §3): N slots, each an input and an output device buffer,
// and three streams - 0 upload, 1 run, 2 download - so that consecutive submissions overlap.  Stream k records a slot's
// event k once the slot's stage k is issued and stream k + 1 waits for it; a slot is taken again only after its
// previous run has read `in` (event 1) and its download has read `out` (event 2), which also guard their regrowth.
// Callers see the run stream and the buffers of the slot they took; streams and events stay in here.
template <int N>
class HostRing {
public:
  HostRing () = default;
  HostRing (const HostRing &) = delete;
  HostRing & operator= (const HostRing &) = delete;

  // the streams and events, once; all or nothing: a failed creation destroys what it made, the next call starts afresh
  cudaError_t setup ()
  {
    if (ready_) return cudaSuccess;
    cudaEvent_t *e = &ev_[0][0];
    cudaError_t err = cudaSuccess;
    int ns = 0, ne = 0;
    while (err == cudaSuccess && ns < 3 && (err = cudaStreamCreateWithFlags (&s_[ns], cudaStreamNonBlocking)) == cudaSuccess) ns++;
    while (err == cudaSuccess && ne < 3 * N && (err = cudaEventCreateWithFlags (&e[ne], cudaEventDisableTiming)) == cudaSuccess) ne++;
    while (err != cudaSuccess && ne > 0) cudaEventDestroy (e[--ne]);
    while (err != cudaSuccess && ns > 0) cudaStreamDestroy (s_[--ns]);
    ready_ = err == cudaSuccess;
    return err;
  }

  // the next slot, its buffers grown to `in_bytes` / `out_bytes` where smaller than `in_need` / `out_need`
  cudaError_t take (size_t in_need = 0, size_t in_bytes = 0, size_t out_need = 0, size_t out_bytes = 0)
  {
    cur_ = submitted_ % N;
    if (used_[cur_]) {
      B200_CUDA_RET (cudaStreamWaitEvent (s_[0], ev_[cur_][1], 0));
      B200_CUDA_RET (cudaStreamWaitEvent (s_[1], ev_[cur_][2], 0));
    }
    B200_CUDA_RET (grow (in_[cur_], 1, in_need, in_bytes));
    return grow (out_[cur_], 2, out_need, out_bytes);
  }
  uint8_t *in (int slot = -1) const { return in_[slot < 0 ? cur_ : slot].ptr; }     // the taken slot's by default
  uint8_t *out (int slot = -1) const { return out_[slot < 0 ? cur_ : slot].ptr; }
  cudaStream_t run_stream () const { return s_[1]; }
  cudaError_t upload (void *dst, const void *src, size_t n) { return cudaMemcpyAsync (dst, src, n, cudaMemcpyHostToDevice, s_[0]); }
  cudaError_t download (void *dst, const void *src, size_t n) { return cudaMemcpyAsync (dst, src, n, cudaMemcpyDeviceToHost, s_[2]); }
  cudaError_t inputs_ready () { return hand_off (0); }      // the run stream waits for the slot's uploads
  cudaError_t run_done () { return hand_off (1); }          // the download stream waits for the slot's device work
  cudaError_t finish ()                                     // the submission is done once its downloads are
  {
    B200_CUDA_RET (cudaEventRecord (ev_[cur_][2], s_[2]));
    used_[cur_] = true; submitted_++;
    return cudaSuccess;
  }

  bool idle (int keep) const { return !ready_ || submitted_ <= (unsigned long long) keep; }
  // all but the `keep` newest submissions back (downloads complete in submission order); only when !idle (keep)
  cudaError_t wait (int keep) { return cudaEventSynchronize (ev_[(submitted_ - 1 - (unsigned long long) keep) % N][2]); }
  // every download (with `uploads`, also every upload no run was ordered after) waited for; the next take is slot 0
  cudaError_t drain (bool uploads = false)
  {
    if (!ready_) return cudaSuccess;
    if (uploads) B200_CUDA_RET (cudaStreamSynchronize (s_[0]));
    B200_CUDA_RET (cudaStreamSynchronize (s_[2]));
    for (int i = 0; i < N; i++) used_[i] = false;
    submitted_ = 0;
    return cudaSuccess;
  }

  // every slot's buffers freed, then allocated at these sizes (cudaFree waits for work still using them)
  cudaError_t resize (size_t in_bytes, size_t out_bytes)
  {
    for (int i = 0; i < N; i++) {
      B200_CUDA_RET (cudaFree (in_[i].ptr)); in_[i] = Buf ();
      B200_CUDA_RET (cudaFree (out_[i].ptr)); out_[i] = Buf ();
    }
    for (int i = 0; i < N; i++) {
      B200_CUDA_RET (cudaMalloc ((void **) &in_[i].ptr, in_bytes)); in_[i].cap = in_bytes;
      B200_CUDA_RET (cudaMalloc ((void **) &out_[i].ptr, out_bytes)); out_[i].cap = out_bytes;
    }
    return cudaSuccess;
  }

  // for the owner's destroy, after drain ()
  void release ()
  {
    if (!ready_) return;
    for (int i = 0; i < N; i++) {
      cudaFree (in_[i].ptr); cudaFree (out_[i].ptr);
      for (int k = 0; k < 3; k++) cudaEventDestroy (ev_[i][k]);
    }
    for (int k = 0; k < 3; k++) cudaStreamDestroy (s_[k]);
  }

private:
  struct Buf { uint8_t *ptr = nullptr; size_t cap = 0; };

  cudaError_t hand_off (int k)
  {
    B200_CUDA_RET (cudaEventRecord (ev_[cur_][k], s_[k]));
    return cudaStreamWaitEvent (s_[k + 1], ev_[cur_][k], 0);
  }
  cudaError_t grow (Buf & b, int guard, size_t need, size_t bytes)
  {
    if (need <= b.cap) return cudaSuccess;
    if (used_[cur_]) B200_CUDA_RET (cudaEventSynchronize (ev_[cur_][guard]));
    B200_CUDA_RET (cudaFree (b.ptr)); b = Buf ();
    B200_CUDA_RET (cudaMalloc ((void **) &b.ptr, bytes));
    b.cap = bytes;
    return cudaSuccess;
  }

  cudaStream_t s_[3] = {};
  cudaEvent_t ev_[N][3] = {};
  Buf in_[N], out_[N];
  bool used_[N] = {}, ready_ = false;
  int cur_ = 0;
  unsigned long long submitted_ = 0;
};

template <typename T>
int upload (T **dptr, const T *host, size_t n)
{
  if (n == 0) { *dptr = nullptr; return B200_OK; }
  B200_CUDA_TRY (cudaMalloc ((void **) dptr, n * sizeof (T)));
  B200_CUDA_TRY (cudaMemcpy (*dptr, host, n * sizeof (T), cudaMemcpyHostToDevice));
  return B200_OK;
}

}  // namespace b200
