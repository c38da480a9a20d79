// gstreamer_b200/csrc/vcs_down420.cuh — chroma down-sampling + 4:2:0 pack (product, sm_90a).
//
// Second launch of the 4:2:0 -> other-4:2:0-family path (NV12 <-> I420, NV12 <-> NV21 ...), which the reference runs
// through its generic chain: after the scalers, chain_downsample (video-converter.c:2018-2032, do_downsample_lines
// :3194-3222) filters the chroma of every line pair (2k, 2k+1) into line 2k, and the pack function of the output
// format (pack_planar_420 video-format.c:117-148, pack_NV12 :1642-1672, pack_NV21 :1818-1848) stores the luma of
// every line and the chroma of the even pixels of the even lines.
//
// The first launch (vcs_generic_kernel with VcsDev::yuv_out) leaves the scaled A,Y,U,V pixels of one frame in a
// scratch image; one thread here produces one chroma sample and the 2x2 luma block under it.
//   vertical   video_chroma_down_v2_u8   (video-chroma.c:434-442; ORC video-orc.orc:2692-2703): avgub of the two lines
//              — V_COSITED selects the reference's unimplemented resampler (:774-785): no vertical filter at all
//   horizontal video_chroma_down_h2_u8   (:398-409; ORC :2657-2671): avgub of the pixel pair
//              video_chroma_down_h2_cs_u8 (:742-764): 3-1 at pixel 0, 1-2-1 inside, 1-3 at the last even pixel >= 2
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200dsp.h"

namespace b200 {

enum Down420H : int { DOWN_H_NONE = 0, DOWN_H_AVG = 1, DOWN_H_COSITED = 2 };

struct Down420Dev {
  int ow, oh;                    // luma size of the output frame
  int stride_s;                  // scratch row pitch in bytes (4 bytes per pixel: A,Y,U,V)
  int hmode, vavg;               // Down420H; 1 = average the line pair
  int extra_row;                 // odd height: the last pair's second line is scratch row `oh` instead of the last line itself
  int stride_y, stride_u, stride_v, cstep;
  unsigned long long off_y, off_u, off_v;
};

struct Down420Batch {
  const uint8_t *scratch[B200_VCS_MAX_BATCH];
  uint8_t *out[B200_VCS_MAX_BATCH];
};

// per-byte (a + b + 1) >> 1 on the U and V bytes (bytes 2 and 3) of two A,Y,U,V words; bytes 0-1 are don't-care
__device__ __forceinline__ unsigned down_avg_uv (unsigned a, unsigned b)
{
  return __vavgu4 (a, b);
}

__global__ void __launch_bounds__ (256)
vcs_down420_kernel (const Down420Dev P, const Down420Batch frames)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;             // chroma column
  const int k = blockIdx.y * blockDim.y + threadIdx.y;             // chroma row
  const int cw = (P.ow + 1) >> 1, chh = (P.oh + 1) >> 1;
  if (j >= cw || k >= chh) return;
  const uint8_t *__restrict__ s = frames.scratch[blockIdx.z];
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const int x0 = 2 * j, y0 = 2 * k;
  const bool two_cols = x0 + 1 < P.ow, two_rows = y0 + 1 < P.oh;
  const unsigned *r0 = (const unsigned *) (s + (size_t) y0 * P.stride_s);
  const unsigned *r1 = (two_rows || P.extra_row) ? (const unsigned *) (s + (size_t) (y0 + 1) * P.stride_s) : r0;

  // the pixels of the pair's two lines this sample reads: x0-1 (co-sited filter only), x0, x0+1
  const unsigned a0 = r0[x0], b0 = r1[x0];
  const unsigned a1 = two_cols ? r0[x0 + 1] : a0, b1 = two_cols ? r1[x0 + 1] : b0;

  // luma: byte 1 of every pixel, every line
  uint8_t *dy = out + P.off_y + (size_t) y0 * P.stride_y + x0;
  dy[0] = (uint8_t) (a0 >> 8);
  if (two_cols) dy[1] = (uint8_t) (a1 >> 8);
  if (two_rows) {
    dy[P.stride_y] = (uint8_t) (b0 >> 8);
    if (two_cols) dy[P.stride_y + 1] = (uint8_t) (b1 >> 8);
  }

  // vertical filter first (it rewrites the whole of line 2k before the horizontal filter runs on it); for an odd
  // height the pair's second line is the vertical scaler's clamped repeat of the last line: avg(a, a) = a — or, with
  // no vertical scaler in the chain, the rebuilt line the first launches left in scratch row `oh` (extra_row)
  const bool vavg = P.vavg != 0;
  const unsigned c0 = vavg ? down_avg_uv (a0, b0) : a0;
  const unsigned c1 = vavg ? down_avg_uv (a1, b1) : a1;
  int u = (c0 >> 16) & 0xff, v = c0 >> 24;
  if (P.hmode == DOWN_H_AVG) {
    if (two_cols) {
      u = (u + (int) ((c1 >> 16) & 0xff) + 1) >> 1;
      v = (v + (int) (c1 >> 24) + 1) >> 1;
    }
  } else if (P.hmode == DOWN_H_COSITED && P.ow >= 2) {
    const int u1 = (c1 >> 16) & 0xff, v1 = c1 >> 24;
    if (x0 == 0) {
      u = (3 * u + u1 + 2) >> 2;                                    // FILT_3_1
      v = (3 * v + v1 + 2) >> 2;
    } else {
      const unsigned am = r0[x0 - 1], bm = r1[x0 - 1];
      const unsigned cm = vavg ? down_avg_uv (am, bm) : am;
      const int um = (cm >> 16) & 0xff, vm = cm >> 24;
      if (x0 < P.ow - 2) {
        u = (um + 2 * u + u1 + 2) >> 2;                             // FILT_1_2_1
        v = (vm + 2 * v + v1 + 2) >> 2;
      } else {
        u = (um + 3 * u + 2) >> 2;                                  // FILT_1_3: the tail pixel of the reference's loop
        v = (vm + 3 * v + 2) >> 2;
      }
    }
  }
  out[P.off_u + (size_t) k * P.stride_u + (size_t) j * P.cstep] = (uint8_t) u;
  out[P.off_v + (size_t) k * P.stride_v + (size_t) j * P.cstep] = (uint8_t) v;
}

// ---- border fill (the element's add-borders): every pixel of every plane outside the destination rectangle takes the
// border value (setup_borderline / convert_fill_border, video-converter.c:2189-2258, :7190-7300)
struct BorderPlane {
  unsigned long long off;
  int stride, pw, ph, bpp;       // plane size in pixels, bytes per pixel (1, 2: interleaved chroma pair, 4: packed RGB)
  int x0, y0, w, h;              // the rectangle in this plane's pixels
  unsigned value;                // pixel bytes, lowest byte first
};
struct BorderDev {
  BorderPlane pl[3];
  int n_planes;
};
struct BorderBatch {
  uint8_t *out[B200_VCS_MAX_BATCH];
};

__global__ void __launch_bounds__ (256)
vcs_border_kernel (const BorderDev P, const BorderBatch frames)
{
  const int plane = blockIdx.z % P.n_planes, frame = blockIdx.z / P.n_planes;
  const BorderPlane & Q = P.pl[plane];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= Q.pw || y >= Q.ph) return;
  if (y >= Q.y0 && y < Q.y0 + Q.h && x >= Q.x0 && x < Q.x0 + Q.w) return;
  uint8_t *d = frames.out[frame] + Q.off + (size_t) y * Q.stride + (size_t) x * Q.bpp;
  if (Q.bpp == 4) {
    d[0] = (uint8_t) Q.value; d[1] = (uint8_t) (Q.value >> 8); d[2] = (uint8_t) (Q.value >> 16); d[3] = (uint8_t) (Q.value >> 24);
  } else if (Q.bpp == 2) {
    d[0] = (uint8_t) Q.value; d[1] = (uint8_t) (Q.value >> 8);
  } else
    d[0] = (uint8_t) Q.value;
}

}  // namespace b200
