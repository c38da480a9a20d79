// gstreamer_b200/csrc/vcs_rgb420.cuh — packed RGB -> 4:2:0: matrix + chroma down-sampling + pack in one pass (product, sm_90a).
//
// The encoder-feeding direction (BGRA / RGBA / ARGB / ABGR and their x forms -> NV12 / NV21 / I420 / YV12) at an unchanged
// or shrinking size.  The reference has no table row for it and runs its chain (video-converter.c:2421-2560): unpack to
// ARGB, every scaler when the frame does not grow (chain_scale :1685-1718), the RGB -> YUV table matrix
// (video_converter_matrix8_table :1178-1200: per component (row . (r,g,b) + offset) >> 8 for a matrix that cannot clip),
// chain_downsample (:2018-2032) on every line pair, pack_NV12 / pack_planar_420.
//
// Product: the scalers are the word-wide plane scaler on 4-byte pixels (vcs_planes_fast.cuh, NC = 4) into a scratch
// image - skipped at an unchanged size, where this kernel reads the input frame itself - and ONE kernel for the rest:
// a thread owns 8 x 2 luma samples (4 chroma samples): two 16-byte loads per line, the matrix as u8 x s8 dot products
// against coefficient words laid out in the source's byte order (each x256 coefficient split into two s8 halves, the
// alpha / padding byte's coefficient 0), the vertical pair average, the horizontal filter of the output's chroma site
// (arithmetic of vcs_down420.cuh, whose header cites the reference's filters), word-wide stores.
// HBM bound: 8 bytes read and 3 bytes written per chroma sample's 2 x 2 block.
// When the frame grows the chain runs the matrix FIRST (chain_scale puts the scalers behind it): vcs_rgb2ayuv_kernel
// (one pixel per thread, the same dot products) leaves A,Y,U,V pixels in a scratch image, the word-wide scaler grows
// them, and this kernel's MATRIX = false form only down-samples and packs.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200dsp.h"
#include "vcs_down420.cuh"

namespace b200 {

struct Rgb420Dev {
  int ow, oh;                    // luma size
  int sstride;                   // source row pitch in bytes (4 bytes per pixel)
  unsigned long long soff;       // byte offset of the source image's first pixel
  int svec;                      // 1: rows are 16-byte aligned, uint4 loads
  unsigned ca[3], cb[3];         // Y, U, V rows: x256 coefficients as two s8 words in the source's byte order (c = a + b)
  int off[3];                    // x256 offsets
  int hmode, vavg;               // Down420H; 1 = average the line pair
  int stride_y, stride_u, stride_v, cstep;
  unsigned long long off_y, off_u, off_v;
  int wvec;                      // 1: every output row is 4-byte aligned, word stores
};

struct Rgb420Batch {
  const uint8_t *src[B200_VCS_MAX_BATCH];
  uint8_t *out[B200_VCS_MAX_BATCH];
};

__device__ __forceinline__ int rgb420_dot (unsigned px, unsigned a, unsigned b, int off)
{
#ifdef B200_CUDA_EMU
  int acc = off;
  for (int k = 0; k < 4; k++)
    acc += (int) ((px >> (8 * k)) & 0xff) * ((int) (int8_t) ((a >> (8 * k)) & 0xff) + (int) (int8_t) ((b >> (8 * k)) & 0xff));
  return acc;
#else
  int d;
  asm ("dp4a.u32.s32 %0, %1, %2, %3;" : "=r" (d) : "r" (px), "r" (a), "r" (off));
  if (b) asm ("dp4a.u32.s32 %0, %1, %2, %0;" : "+r" (d) : "r" (px), "r" (b));
  return d;
#endif
}

// one line's 8 pixels (+ the one before them) -> 8 luma bytes and the U / V bytes of pixels -1 .. 7 (byte lanes of uq / vq words)
struct Rgb420Line {
  unsigned y[2];                 // luma of pixels 0-3, 4-7
  unsigned u[2], v[2];           // chroma of pixels 0-3, 4-7
  unsigned um, vm;               // chroma of the pixel left of the block (co-sited filter), in byte 0
};

template <bool MATRIX>
__device__ __forceinline__ void rgb420_line (const Rgb420Dev & P, const uint8_t * __restrict__ row, int x0, bool full, bool left, Rgb420Line & L)
{
  unsigned px[8];
  if (full && P.svec) {
    const uint4 q0 = __ldg ((const uint4 *) (row + (size_t) x0 * 4)), q1 = __ldg ((const uint4 *) (row + (size_t) x0 * 4 + 16));
    px[0] = q0.x; px[1] = q0.y; px[2] = q0.z; px[3] = q0.w; px[4] = q1.x; px[5] = q1.y; px[6] = q1.z; px[7] = q1.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++) px[i] = __ldg ((const unsigned *) row + min (x0 + i, P.ow - 1));
  }
  L.y[0] = L.y[1] = L.u[0] = L.u[1] = L.v[0] = L.v[1] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    unsigned yy, uu, vv;
    if (MATRIX) {
      yy = (unsigned) (rgb420_dot (px[i], P.ca[0], P.cb[0], P.off[0]) >> 8) & 0xff;
      uu = (unsigned) (rgb420_dot (px[i], P.ca[1], P.cb[1], P.off[1]) >> 8) & 0xff;
      vv = (unsigned) (rgb420_dot (px[i], P.ca[2], P.cb[2], P.off[2]) >> 8) & 0xff;
    } else {                                                        // A,Y,U,V pixels of vcs_rgb2ayuv_kernel
      yy = (px[i] >> 8) & 0xff; uu = (px[i] >> 16) & 0xff; vv = px[i] >> 24;
    }
    L.y[i >> 2] |= yy << (8 * (i & 3));
    L.u[i >> 2] |= uu << (8 * (i & 3));
    L.v[i >> 2] |= vv << (8 * (i & 3));
  }
  L.um = L.vm = 0;
  if (left) {
    const unsigned pm = __ldg ((const unsigned *) row + (x0 - 1));
    if (MATRIX) {
      L.um = (unsigned) (rgb420_dot (pm, P.ca[1], P.cb[1], P.off[1]) >> 8) & 0xff;
      L.vm = (unsigned) (rgb420_dot (pm, P.ca[2], P.cb[2], P.off[2]) >> 8) & 0xff;
    } else {
      L.um = (pm >> 16) & 0xff; L.vm = pm >> 24;
    }
  }
}

// horizontal chroma filter of one component: c[0..1] hold the (vertically filtered) samples of pixels 0-7, cm pixel -1;
// returns the 4 chroma samples of the even pixels as one word.  x0: first pixel of the block
__device__ __forceinline__ unsigned rgb420_down_h (const Rgb420Dev & P, const unsigned c[2], unsigned cm, int x0)
{
  unsigned o = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int x = x0 + 2 * j;
    const int cur = (c[j >> 1] >> (16 * (j & 1))) & 0xff;
    const int nxt = (c[j >> 1] >> (16 * (j & 1) + 8)) & 0xff;
    int r = cur;
    if (P.hmode == DOWN_H_AVG) {
      if (x + 1 < P.ow) r = (cur + nxt + 1) >> 1;
    } else if (P.hmode == DOWN_H_COSITED && P.ow >= 2) {
      const int prv = j == 0 ? (int) cm : (int) ((c[(j - 1) >> 1] >> (16 * ((j - 1) & 1) + 8)) & 0xff);
      if (x == 0) r = (3 * cur + nxt + 2) >> 2;                     // FILT_3_1
      else if (x < P.ow - 2) r = (prv + 2 * cur + nxt + 2) >> 2;   // FILT_1_2_1
      else r = (prv + 3 * cur + 2) >> 2;                           // FILT_1_3
    }
    o |= (unsigned) r << (8 * j);
  }
  return o;
}

template <bool MATRIX>
__global__ void __launch_bounds__ (256)
vcs_rgb420_kernel (const Rgb420Dev P, const Rgb420Batch frames)
{
  const int jb = blockIdx.x * blockDim.x + threadIdx.x;            // block of 4 chroma columns
  const int k = blockIdx.y * blockDim.y + threadIdx.y;             // chroma row
  const int cw = (P.ow + 1) >> 1, chh = (P.oh + 1) >> 1;
  if (4 * jb >= cw || k >= chh) return;
  const uint8_t *__restrict__ s = frames.src[blockIdx.z] + P.soff;
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const int x0 = 8 * jb, y0 = 2 * k;
  const bool full = x0 + 8 <= P.ow, two_rows = y0 + 1 < P.oh;
  const bool left = P.hmode == DOWN_H_COSITED && x0 > 0;

  Rgb420Line A, B;
  rgb420_line<MATRIX> (P, s + (size_t) y0 * P.sstride, x0, full, left, A);
  if (two_rows) rgb420_line<MATRIX> (P, s + (size_t) (y0 + 1) * P.sstride, x0, full, left, B);
  else B = A;                                                       // odd height: the pair's second line is the last line itself

  // luma: every pixel of both lines
  uint8_t *dy = out + P.off_y + (size_t) y0 * P.stride_y + x0;
  if (full && P.wvec) {
    ((unsigned *) dy)[0] = A.y[0]; ((unsigned *) dy)[1] = A.y[1];
    if (two_rows) { ((unsigned *) (dy + P.stride_y))[0] = B.y[0]; ((unsigned *) (dy + P.stride_y))[1] = B.y[1]; }
  } else {
    for (int i = 0; i < 8 && x0 + i < P.ow; i++) {
      dy[i] = (uint8_t) (A.y[i >> 2] >> (8 * (i & 3)));
      if (two_rows) dy[P.stride_y + i] = (uint8_t) (B.y[i >> 2] >> (8 * (i & 3)));
    }
  }

  // chroma: vertical filter first (chain_downsample rewrites the whole of line 2k before the horizontal filter runs on it)
  unsigned cu[2], cv[2], um = A.um, vm = A.vm;
  cu[0] = A.u[0]; cu[1] = A.u[1]; cv[0] = A.v[0]; cv[1] = A.v[1];
  if (P.vavg) {
    cu[0] = __vavgu4 (A.u[0], B.u[0]); cu[1] = __vavgu4 (A.u[1], B.u[1]);
    cv[0] = __vavgu4 (A.v[0], B.v[0]); cv[1] = __vavgu4 (A.v[1], B.v[1]);
    um = __vavgu4 (A.um, B.um); vm = __vavgu4 (A.vm, B.vm);
  }
  const unsigned ou = rgb420_down_h (P, cu, um, x0), ov = rgb420_down_h (P, cv, vm, x0);
  const bool cfull = 4 * jb + 4 <= cw;
  if (P.cstep == 1) {
    uint8_t *du = out + P.off_u + (size_t) k * P.stride_u + 4 * jb, *dv = out + P.off_v + (size_t) k * P.stride_v + 4 * jb;
    if (cfull && P.wvec) { *(unsigned *) du = ou; *(unsigned *) dv = ov; }
    else for (int j = 0; j < 4 && 4 * jb + j < cw; j++) { du[j] = (uint8_t) (ou >> (8 * j)); dv[j] = (uint8_t) (ov >> (8 * j)); }
  } else {                                                          // interleaved pairs: U first (NV12) or V first (NV21)
    const bool v_first = P.off_v < P.off_u;
    const unsigned e = v_first ? ov : ou, o = v_first ? ou : ov;
    uint8_t *dc = out + (v_first ? P.off_v : P.off_u) + (size_t) k * P.stride_u + 8 * jb;
    if (cfull && P.wvec) {
      ((unsigned *) dc)[0] = __byte_perm (e, o, 0x5140);
      ((unsigned *) dc)[1] = __byte_perm (e, o, 0x7362);
    } else
      for (int j = 0; j < 4 && 4 * jb + j < cw; j++) { dc[2 * j] = (uint8_t) (e >> (8 * j)); dc[2 * j + 1] = (uint8_t) (o >> (8 * j)); }
  }
}

// coefficient words of one matrix row for a source whose R, G, B bytes sit at byte positions pos_r / pos_g / pos_b
inline bool rgb420_split_row (const int row[4], int pos_r, int pos_g, int pos_b, unsigned * a, unsigned * b)
{
  const int pos[3] = {pos_r, pos_g, pos_b};
  *a = *b = 0;
  for (int i = 0; i < 3; i++) {
    const int c = row[i];
    if (c < -256 || c > 254) return false;
    const int ca = c > 127 ? 127 : (c < -128 ? -128 : c), cb = c - ca;
    *a |= (unsigned) (uint8_t) (int8_t) ca << (8 * pos[i]);
    *b |= (unsigned) (uint8_t) (int8_t) cb << (8 * pos[i]);
  }
  return true;
}

// the matrix alone: packed RGB pixels -> A,Y,U,V pixels (bytes 0..3) of the same size, one pixel per thread
struct Rgb2AyuvDev {
  int w, h;
  int sstride, dstride;          // bytes
  unsigned long long soff;
  unsigned ca[3], cb[3];
  int off[3];
};

__global__ void __launch_bounds__ (256)
vcs_rgb2ayuv_kernel (const Rgb2AyuvDev P, const Rgb420Batch frames)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= P.w) return;
  const unsigned px = __ldg ((const unsigned *) (frames.src[blockIdx.z] + P.soff + (size_t) y * P.sstride) + x);
  const unsigned yy = (unsigned) (rgb420_dot (px, P.ca[0], P.cb[0], P.off[0]) >> 8) & 0xff;
  const unsigned uu = (unsigned) (rgb420_dot (px, P.ca[1], P.cb[1], P.off[1]) >> 8) & 0xff;
  const unsigned vv = (unsigned) (rgb420_dot (px, P.ca[2], P.cb[2], P.off[2]) >> 8) & 0xff;
  ((unsigned *) (frames.out[blockIdx.z] + (size_t) y * P.dstride))[x] = 0xffu | (yy << 8) | (uu << 16) | (vv << 24);
}

inline int launch_rgb2ayuv (const Rgb2AyuvDev & d, const Rgb420Batch & batch, int n, cudaStream_t stream)
{
  dim3 grid ((d.w + 255) / 256, d.h, n);
  vcs_rgb2ayuv_kernel <<<grid, 256, 0, stream>>> (d, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

// packed 4:2:2 (YUY2 / UYVY / YVYU) -> A,Y,U,V pixels of the same size: unpack (each pair's chroma sample feeds both pixels,
// video-format.c:155-274) + the 4:2:2 horizontal chroma up-sampler of the input's site, one pixel per thread.
//   co-sited  video_chroma_up_h2_cs_u8 (video-chroma.c:687-699): odd pixels x <= w - 2 take (c[k] + c[k+1] + 1) >> 1
//   centred   video_chroma_up_h2_u8 (:309-327): pixel 0 keeps c[0]; odd x <= w - 2: (3 c[k] + c[k+1] + 2) >> 2;
//             even x >= 2: (c[k-1] + 3 c[k] + 2) >> 2; a last odd pixel x = w - 1 keeps c[k]        (k = x >> 1)
struct Yuy2AyuvDev {
  int w, h;
  int sstride, dstride;
  unsigned long long soff;
  int ypos, upos, vpos;          // byte of Y0, U, V inside a pixel pair's word (Y1 = ypos + 2)
  int cosited;
};

__global__ void __launch_bounds__ (256)
vcs_yuy2_ayuv_kernel (const Yuy2AyuvDev P, const Rgb420Batch frames)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= P.w) return;
  const unsigned *row = (const unsigned *) (frames.src[blockIdx.z] + P.soff + (size_t) y * P.sstride);
  const int k = x >> 1, np = (P.w + 1) >> 1;
  const unsigned own = __ldg (row + k);
  const unsigned yy = (own >> (8 * (P.ypos + 2 * (x & 1)))) & 0xff;
  unsigned u = (own >> (8 * P.upos)) & 0xff, v = (own >> (8 * P.vpos)) & 0xff;
  if ((x & 1) && x < P.w - 1) {                                    // odd pixel with a pair to its right
    const unsigned nb = __ldg (row + min (k + 1, np - 1));
    const unsigned un = (nb >> (8 * P.upos)) & 0xff, vn = (nb >> (8 * P.vpos)) & 0xff;
    if (P.cosited) { u = (u + un + 1) >> 1; v = (v + vn + 1) >> 1; }
    else { u = (3 * u + un + 2) >> 2; v = (3 * v + vn + 2) >> 2; }
  } else if (!(x & 1) && x >= 2 && !P.cosited) {                   // even pixel behind another pair (centred site only)
    const unsigned nb = __ldg (row + (k - 1));
    const unsigned up = (nb >> (8 * P.upos)) & 0xff, vp = (nb >> (8 * P.vpos)) & 0xff;
    u = (up + 3 * u + 2) >> 2; v = (vp + 3 * v + 2) >> 2;
  }
  ((unsigned *) (frames.out[blockIdx.z] + (size_t) y * P.dstride))[x] = 0xffu | (yy << 8) | (u << 16) | (v << 24);
}

inline int launch_yuy2_ayuv (const Yuy2AyuvDev & d, const Rgb420Batch & batch, int n, cudaStream_t stream)
{
  dim3 grid ((d.w + 255) / 256, d.h, n);
  vcs_yuy2_ayuv_kernel <<<grid, 256, 0, stream>>> (d, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

inline int launch_rgb420 (const Rgb420Dev & d, const Rgb420Batch & batch, int n, cudaStream_t stream, bool matrix = true)
{
  const int cw = (d.ow + 1) / 2, chh = (d.oh + 1) / 2, cb = (cw + 3) / 4;
  dim3 blk (32, 8), grid ((cb + 31) / 32, (chh + 7) / 8, n);
  if (matrix) vcs_rgb420_kernel<true> <<<grid, blk, 0, stream>>> (d, batch);
  else vcs_rgb420_kernel<false> <<<grid, blk, 0, stream>>> (d, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
