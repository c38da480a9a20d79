// gstreamer_b200/csrc/vcs_yuy2_420.cuh — packed 4:2:2 -> planar 4:2:0 at an unchanged size (product, sm_90a).
//
// The capture -> encoder rows of the reference's fast-path table (video-converter.c:8493-8507): YUY2 / UYVY -> I420 / YV12,
// unchanged size, same colour matrix (range and chroma-site are not looked at, :8985-8997; a border rectangle or any other
// pair takes the chain instead).  convert_YUY2_I420 / convert_UYVY_I420 (:3954-4028, :4913-4986) run
// video_orc_convert_YUY2_I420 / _UYVY_I420 (video-orc.orc:716-744, :781-809) on every line pair: the luma of both lines is
// copied - (width + 1) / 2 PAIRS, so an odd width also writes one byte of row padding - and each chroma sample is avgub of
// the pair's two lines, no horizontal filter.  A last odd line goes through unpack + pack_planar_420 (video-format.c:117-148):
// exactly `width` luma bytes, its own chroma.
//
// One thread = 8 x 2 luma samples: one 16-byte load per line, PRMT de-interleave, __vavgu4, word stores.
// HBM bound: 4 bytes read and 3 written per 2 x 1 pixel pair of a line pair.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200dsp.h"
#include "common.h"

namespace b200 {

struct Yuy2Dev {
  int w, h;
  int sstride;
  unsigned long long soff;
  unsigned sel_y, sel_c;         // PRMT selectors over two source words: the 4 luma bytes / (U, V, U, V) of two pixel pairs
  int svec;                      // 2: rows 16-byte aligned (LDG.128), 1: 4-byte aligned (LDG.32), 0: byte loads
  int stride_y, stride_u, stride_v;
  unsigned long long off_y, off_u, off_v;
  int wvec;                      // 1: output rows 4-byte aligned, word stores
};

struct Yuy2Batch {
  const uint8_t *src[B200_VCS_MAX_BATCH];
  uint8_t *out[B200_VCS_MAX_BATCH];
};

// one line's 4 source words (8 pixels) starting at pixel pair `pair0`; pairs past the line's (w + 1) / 2 repeat the last one
__device__ __forceinline__ void yuy2_line (const Yuy2Dev & P, const uint8_t * __restrict__ row, int pair0, int np, bool full,
    unsigned (&yw)[2], unsigned & u, unsigned & v)
{
  unsigned w[4];
  if (full && P.svec == 2) {
    const uint4 q = __ldg ((const uint4 *) (row + (size_t) pair0 * 4));
    w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w;
  } else {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint8_t *p = row + (size_t) min (pair0 + i, np - 1) * 4;
      if (P.svec) w[i] = __ldg ((const unsigned *) p);
      else w[i] = (unsigned) p[0] | ((unsigned) p[1] << 8) | ((unsigned) p[2] << 16) | ((unsigned) p[3] << 24);
    }
  }
  yw[0] = __byte_perm (w[0], w[1], P.sel_y); yw[1] = __byte_perm (w[2], w[3], P.sel_y);
  const unsigned c01 = __byte_perm (w[0], w[1], P.sel_c), c23 = __byte_perm (w[2], w[3], P.sel_c);   // U V U V
  u = __byte_perm (c01, c23, 0x6420); v = __byte_perm (c01, c23, 0x7531);
}

__global__ void __launch_bounds__ (256)
vcs_yuy2_420_kernel (const Yuy2Dev P, const Yuy2Batch frames)
{
  const int jb = blockIdx.x * blockDim.x + threadIdx.x;            // block of 4 pixel pairs
  const int k = blockIdx.y * blockDim.y + threadIdx.y;             // chroma row
  const int np = (P.w + 1) >> 1, chh = (P.h + 1) >> 1;
  if (4 * jb >= np || k >= chh) return;
  const uint8_t *__restrict__ s = frames.src[blockIdx.z] + P.soff;
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const int y0 = 2 * k;
  const bool two_rows = y0 + 1 < P.h, full = 4 * jb + 4 <= np;
  unsigned ya[2], yb[2], ua, va, ub, vb;
  yuy2_line (P, s + (size_t) y0 * P.sstride, 4 * jb, np, full, ya, ua, va);
  if (two_rows) yuy2_line (P, s + (size_t) (y0 + 1) * P.sstride, 4 * jb, np, full, yb, ub, vb);
  else { yb[0] = ya[0]; yb[1] = ya[1]; ub = ua; vb = va; }

  // luma: whole pairs on a line pair (an odd width spills one byte into the row padding, like the reference), exactly
  // `w` bytes on a last odd line
  uint8_t *dy = out + P.off_y + (size_t) y0 * P.stride_y + 8 * jb;
  const int ny = min ((two_rows ? 2 * np : P.w) - 8 * jb, 8);
  if (ny == 8 && P.wvec) {
    ((unsigned *) dy)[0] = ya[0]; ((unsigned *) dy)[1] = ya[1];
    if (two_rows) { ((unsigned *) (dy + P.stride_y))[0] = yb[0]; ((unsigned *) (dy + P.stride_y))[1] = yb[1]; }
  } else {
    for (int i = 0; i < ny; i++) {
      dy[i] = (uint8_t) (ya[i >> 2] >> (8 * (i & 3)));
      if (two_rows) dy[P.stride_y + i] = (uint8_t) (yb[i >> 2] >> (8 * (i & 3)));
    }
  }
  const unsigned ou = __vavgu4 (ua, ub), ov = __vavgu4 (va, vb);  // avgub of the two lines; a last odd line averages with itself
  uint8_t *du = out + P.off_u + (size_t) k * P.stride_u + 4 * jb, *dv = out + P.off_v + (size_t) k * P.stride_v + 4 * jb;
  if (full && P.wvec) { *(unsigned *) du = ou; *(unsigned *) dv = ov; }
  else for (int j = 0; j < 4 && 4 * jb + j < np; j++) { du[j] = (uint8_t) (ou >> (8 * j)); dv[j] = (uint8_t) (ov >> (8 * j)); }
}

inline int launch_yuy2_420 (const Yuy2Dev & d, const Yuy2Batch & batch, int n, cudaStream_t stream)
{
  const int np = (d.w + 1) / 2, chh = (d.h + 1) / 2, cb = (np + 3) / 4;
  dim3 blk (32, 8), grid ((cb + 31) / 32, (chh + 7) / 8, n);
  vcs_yuy2_420_kernel <<<grid, blk, 0, stream>>> (d, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
