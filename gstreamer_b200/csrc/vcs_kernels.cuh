// gstreamer_b200/csrc/vcs_kernels.cuh — convert+scale device code (product, sm_90a).
//
// Integer arithmetic here reproduces, stage by stage, what the reference's ORC
// programs compute (gst-libs/gst/video/video-orc.orc); each helper cites its program.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "vcs_device.h"

namespace b200 {

// (acc + 32) >> 6 in wrapping 16-bit, then saturate to u8
// video_orc_resample_scaletaps_u8_lq, video-orc.orc:2474-2481 (addw 32; shrsw 6; convsuswb)
__device__ __forceinline__ int fir_round_u8 (int acc)
{
  int v = ((int) (short) (acc + 32)) >> 6;
  return min (max (v, 0), 255);
}

// d = s0 + hi8((s1 - s0) * p1 + 128) in wrapping 16/8-bit
// video_orc_resample_v_2tap_u8_lq, video-orc.orc:2212-2228
__device__ __forceinline__ int lerp_v_u8 (int s0, int s1, int p1)
{
  int w = (int) (short) ((short) (s1 - s0) * p1);
  w = (w + 128) & 0xffff;
  return (s0 + (w >> 8)) & 0xff;
}

// (a*(256-f) + b*f) >> 8 : ldreslinl, C semantics in video-orc-dist.c video_orc_resample_h_2tap_4u8_lq
__device__ __forceinline__ int lerp_h_u8 (int a, int b, int f)
{
  return (a * (256 - f) + b * f) >> 8;
}

// One chroma component of one chroma row, horizontally upsampled to luma column x.
// cosited:      video_chroma_up_h2_cs_u8, video-chroma.c:687-699
// non-cosited:  video_chroma_up_h2_u8,    video-chroma.c:277-296
// mode 2 (nearest): no filter at all — unpack's replication (loadupdb), what the I420 fast path keeps
// c points at sample 0 of that component in its chroma row; consecutive samples are `step` bytes apart
// (2 in an interleaved UV row, 1 in a planar one).
__device__ __forceinline__ int chroma_hup (const uint8_t * __restrict__ c, int x, int iw, int mode, int step = 2)
{
  if (mode == 3)                 // 4:4:4: every pixel has its own sample, no filter (no chroma resampler exists)
    return c[step * x];
  const int k = x >> 1;
  if (mode == 2)
    return c[step * k];
  if (mode == 1) {
    if ((x & 1) && x < iw - 1)
      return (c[step * k] + c[step * k + step] + 1) >> 1;
    return c[step * k];
  }
  if (x == 0 || ((x & 1) && x >= iw - 1))
    return c[step * k];
  if (x & 1)
    return (3 * c[step * k] + c[step * k + step] + 2) >> 2;
  return (c[step * k - step] + 3 * c[step * k] + 2) >> 2;
}

// video_orc_convert_AYUV_ARGB, video-orc.orc:1634-1688:
//   x -= 128 (bytes); w = splatbw(x); t = mulhsw(w, p); sums in 16 bit; convssswb; += 128
// splatbw of the biased byte ub=(x^0x80) read as s16 is (x-128)*256 + ub.
__device__ __forceinline__ int splat_s16 (int x)
{
  return (x - 128) * 256 + (x ^ 0x80);
}

__device__ __forceinline__ void yuv_to_rgb (int y, int u, int v, int p1, int p2, int p3, int p4, int p5,
    int &r, int &g, int &b)
{
  const int wy = (splat_s16 (y) * p1) >> 16;
  const int wu = splat_s16 (u), wv = splat_s16 (v);
  int rr = wy + ((wv * p2) >> 16);
  int bb = wy + ((wu * p3) >> 16);
  int gg = wy + ((wu * p4) >> 16) + ((wv * p5) >> 16);
  // addw wraps at 16 bit before convssswb; |sum| stays far below 2^15 for 8-bit input and
  // |p| < 2^15, so the wrap is a no-op and only the signed-byte saturation remains.
  r = min (max (rr, -128), 127) + 128;
  g = min (max (gg, -128), 127) + 128;
  b = min (max (bb, -128), 127) + 128;
}

// video_converter_matrix8_table (video-converter.c:1178-1200; tables :1110-1134): for a matrix that cannot clip
// (is_no_clip_matrix :1262-1300) the three 16-bit fields of its packed 64-bit sums never borrow from each other, so
// each component is (row . (r,g,b) + offset) >> 8
__device__ __forceinline__ void rgb_to_yuv (int r, int g, int b, const int (&m)[3][4], int &y, int &u, int &v)
{
  y = (m[0][0] * r + m[0][1] * g + m[0][2] * b + m[0][3]) >> 8;
  u = (m[1][0] * r + m[1][1] * g + m[1][2] * b + m[1][3]) >> 8;
  v = (m[2][0] * r + m[2][1] * g + m[2][2] * b + m[2][3]) >> 8;
}

// alpha travels through the scalers as a constant 255 line (unpack sets A=0xff,
// video-format.c:1612-1637): n-tap passes turn it into round(255 * sum(taps)).
__device__ __forceinline__ int alpha_pass (int a, const AxisDev & ax, int idx)
{
  if (ax.mode == 3)
    return fir_round_u8 ((int) (short) (a * (int) ax.sum[idx]));
  return a;
}

__device__ __forceinline__ unsigned pack_px (int a, int r, int g, int b, unsigned sel)
{
  // comp index 0..3 = A,R,G,B ; byte i of the output word takes comp (sel >> 4i) & 3
  const unsigned argb = (unsigned) a | ((unsigned) r << 8) | ((unsigned) g << 16) | ((unsigned) b << 24);
  return __byte_perm (argb, 0, sel);
}

// planar RGB store form (RGBP / BGRP): bytes 0..2 of the packed pixel `px` (the plan's byte selector is that of RGBx /
// BGRx) go to planes 0..2.  A lane owns one output column, so a warp's byte stores to a plane row are consecutive.
__device__ __forceinline__ void store_planar_px (const VcsDev & P, uint8_t *out, int ox, int oy, unsigned px)
{
  out[P.off_pl[0] + (size_t) oy * P.stride_pl[0] + ox] = (uint8_t) px;
  out[P.off_pl[1] + (size_t) oy * P.stride_pl[1] + ox] = (uint8_t) (px >> 8);
  out[P.off_pl[2] + (size_t) oy * P.stride_pl[2] + ox] = (uint8_t) (px >> 16);
}

// ------------------------------------------------------------------------------------------
// Generic fused kernel: one CTA = one output tile of one frame.
//   A1  h-upsampled chroma rows of the tile's input region  -> smem
//   A2  Y + v-combined chroma (optionally -> RGB)           -> smem planes S[3]
//   B   first separable pass                                -> smem planes T[3]
//   C   second pass + matrix + alpha + pack                 -> global (coalesced 4 B / thread)
// Handles every scale method / ratio / order the plan builder can emit.
// PLOUT: planar RGB output (store_planar_px) instead of one 4-byte word per pixel.
// ------------------------------------------------------------------------------------------
template <bool PLOUT = false>
__global__ void __launch_bounds__ (256)
vcs_generic_kernel (const VcsDev P, const VcsBatch frames)
{
  extern __shared__ __align__ (16) uint8_t smem[];
  const int tid = threadIdx.x, nthr = blockDim.x;
  const uint8_t *__restrict__ in = frames.in[blockIdx.z];
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const uint8_t *__restrict__ plane_y = in + P.off_y;

  const int ox0 = blockIdx.x * P.tile_w, oy0 = blockIdx.y * P.tile_h;
  const int tw = min (P.tile_w, P.ow - ox0), th = min (P.tile_h, P.oh - oy0);
  const int cx0 = P.h.offset[ox0], cx1 = P.h.offset[ox0 + tw - 1] + P.h.span;   // input cols [cx0,cx1)
  const int ry0 = P.v.offset[oy0], ry1 = P.v.offset[oy0 + th - 1] + P.v.span;   // input rows [ry0,ry1)
  const int R = ry1 - ry0, C = cx1 - cx0, Cp = P.cols_pitch;

  // shared memory carve-up (sizes from the plan's maxima)
  uint8_t *S = smem;                                            // [3][max_rows][Cp]
  const int plane_sz = P.max_rows * Cp;
  uint8_t *HU = S + 3 * plane_sz;                               // [2][max_crows][Cp]
  const int hup_sz = P.max_crows * Cp;
  uint8_t *T = HU + 2 * hup_sz;                                 // h_first: [3][max_rows][tile_w]; else [3][tile_h][Cp]
  const int mid_sz = P.h_first ? P.max_rows * P.tile_w : P.tile_h * Cp;
  int16_t *CH = (int16_t *) (((uintptr_t) (T + 3 * mid_sz) + 15) & ~(uintptr_t) 15);   // [tile_w][coef_per_out]
  int16_t *CV = CH + P.tile_w * max (P.h.coef_per_out, 1);                                // [tile_h][coef_per_out]

  // stage the tile's coefficients
  for (int i = tid; i < tw * P.h.coef_per_out; i += nthr)
    CH[i] = P.h.coef[(size_t) ox0 * P.h.coef_per_out + i];
  for (int i = tid; i < th * P.v.coef_per_out; i += nthr)
    CV[i] = P.v.coef[(size_t) oy0 * P.v.coef_per_out + i];

  // ---- A1: chroma rows, horizontally upsampled to the region's columns
  // chroma rows the tile touches (inclusive): with 4:2:0 the rows of the lines one above / below too (line pairs)
  const int cr0 = P.cvshift ? max (ry0 - 1, 0) >> 1 : ry0, cr1 = P.cvshift ? min (ry1, P.ih - 1) >> 1 : ry1 - 1;
  const int ncr = cr1 - cr0 + 1;
  for (int i = tid; i < (P.rgb_in ? 0 : ncr * C); i += nthr) {
    const int r = i / C, c = i - r * C;
    const int x = cx0 + c;
    const int hmode = P.chshift == 0 ? 3 : (P.chroma_nearest ? 2 : P.h_cosited);
    HU[r * Cp + c] = (uint8_t) chroma_hup (in + P.off_u + (size_t) (cr0 + r) * P.stride_u, x, P.iw, hmode, P.cstep);
    HU[hup_sz + r * Cp + c] = (uint8_t) chroma_hup (in + P.off_v + (size_t) (cr0 + r) * P.stride_v, x, P.iw, hmode, P.cstep);
  }
  __syncthreads ();

  // ---- A2: luma + vertically combined chroma (pairing decided per line by the plan)
  for (int i = tid; i < R * C; i += nthr) {
    const int r = i / C, c = i - r * C;
    const int y = ry0 + r;
    const int own = (y >> P.cvshift) - cr0;
    int yy, u, v;
    if (P.rgb_in) {
      // unpack_BGRA / _RGBA / _ABGR / unpack_copy4 (video-format.c:1433-1502, :536-547): a byte shuffle to A,R,G,B
      const unsigned px = __byte_perm (*(const unsigned *) (plane_y + (size_t) y * P.stride_y + 4 * (size_t) (cx0 + c)), 0, P.in_sel);
      yy = px & 0xff; u = (px >> 8) & 0xff; v = (px >> 16) & 0xff;
      if (P.matrix_first) rgb_to_yuv (yy, u, v, P.m, yy, u, v);
      S[r * Cp + c] = (uint8_t) yy;
      S[plane_sz + r * Cp + c] = (uint8_t) u;
      S[2 * plane_sz + r * Cp + c] = (uint8_t) v;
      continue;
    }
    yy = plane_y[(size_t) y * P.stride_y + (size_t) (cx0 + c) * P.ystep];
    u = HU[own * Cp + c]; v = HU[hup_sz + own * Cp + c];
    const int m = P.v_pairs ? P.chroma_mode[y] : 0;
    if (m) {
      const int oth = ((m == 1 ? min (y + 1, P.ih - 1) : y - 1) >> 1) - cr0;
      u = (3 * u + HU[oth * Cp + c] + 2) >> 2;                    // FILT_3_1 / FILT_1_3, video-chroma.c:255-256
      v = (3 * v + HU[hup_sz + oth * Cp + c] + 2) >> 2;
    }
    if (P.matrix_first) {
      int rr, gg, bb;
      yuv_to_rgb (yy, u, v, P.p1, P.p2, P.p3, P.p4, P.p5, rr, gg, bb);
      yy = rr; u = gg; v = bb;
    }
    S[r * Cp + c] = (uint8_t) yy;
    S[plane_sz + r * Cp + c] = (uint8_t) u;
    S[2 * plane_sz + r * Cp + c] = (uint8_t) v;
  }
  __syncthreads ();

  // ---- B: first pass
  if (P.h_first) {
    for (int i = tid; i < R * tw; i += nthr) {
      const int r = i / tw, tx = i - r * tw;
      const int base = (int) P.h.offset[ox0 + tx] - cx0;
#pragma unroll
      for (int ch = 0; ch < 3; ch++) {
        const uint8_t *s = S + ch * plane_sz + r * Cp + base;
        int val;
        if (P.h.mode == 1) val = s[0];
        else if (P.h.mode == 2) val = lerp_h_u8 (s[0], s[1], CH[tx]);
        else {
          const int16_t *t = CH + tx * P.h.n_taps;
          int acc = 0;
          for (int k = 0; k < P.h.n_taps; k++) acc += (int) s[k] * (int) t[k];
          val = fir_round_u8 (acc);
        }
        T[ch * mid_sz + r * P.tile_w + tx] = (uint8_t) val;
      }
    }
  } else {
    for (int i = tid; i < th * C; i += nthr) {
      const int ty = i / C, c = i - ty * C;
      const int base = (int) P.v.offset[oy0 + ty] - ry0;
#pragma unroll
      for (int ch = 0; ch < 3; ch++) {
        const uint8_t *s = S + ch * plane_sz + base * Cp + c;
        int val;
        if (P.v.mode == 1) val = s[0];
        else if (P.v.mode == 2) val = lerp_v_u8 (s[0], s[Cp], CV[ty]);
        else {
          const int16_t *t = CV + ty * P.v.n_taps;
          int acc = 0;
          for (int k = 0; k < P.v.n_taps; k++) acc += (int) s[k * Cp] * (int) t[k];
          val = fir_round_u8 (acc);
        }
        T[ch * mid_sz + ty * Cp + c] = (uint8_t) val;
      }
    }
  }
  __syncthreads ();

  // ---- C: second pass, matrix, alpha, pack, store
  for (int i = tid; i < th * tw; i += nthr) {
    const int ty = i / tw, tx = i - ty * tw;
    const int ox = ox0 + tx, oy = oy0 + ty;
    int comp[3];
    if (P.h_first) {
      const int base = (int) P.v.offset[oy] - ry0;
#pragma unroll
      for (int ch = 0; ch < 3; ch++) {
        const uint8_t *s = T + ch * mid_sz + base * P.tile_w + tx;
        if (P.v.mode == 1) comp[ch] = s[0];
        else if (P.v.mode == 2) comp[ch] = lerp_v_u8 (s[0], s[P.tile_w], CV[ty]);
        else {
          const int16_t *t = CV + ty * P.v.n_taps;
          int acc = 0;
          for (int k = 0; k < P.v.n_taps; k++) acc += (int) s[k * P.tile_w] * (int) t[k];
          comp[ch] = fir_round_u8 (acc);
        }
      }
    } else {
      const int base = (int) P.h.offset[ox] - cx0;
#pragma unroll
      for (int ch = 0; ch < 3; ch++) {
        const uint8_t *s = T + ch * mid_sz + ty * Cp + base;
        if (P.h.mode == 1) comp[ch] = s[0];
        else if (P.h.mode == 2) comp[ch] = lerp_h_u8 (s[0], s[1], CH[tx]);
        else {
          const int16_t *t = CH + tx * P.h.n_taps;
          int acc = 0;
          for (int k = 0; k < P.h.n_taps; k++) acc += (int) s[k] * (int) t[k];
          comp[ch] = fir_round_u8 (acc);
        }
      }
    }
    int r, g, b;
    if (P.rgb_in && !P.matrix_first) rgb_to_yuv (comp[0], comp[1], comp[2], P.m, r, g, b);
    else if (P.matrix_first || P.yuv_out) { r = comp[0]; g = comp[1]; b = comp[2]; }
    else yuv_to_rgb (comp[0], comp[1], comp[2], P.p1, P.p2, P.p3, P.p4, P.p5, r, g, b);
    int a = 255;
    if (P.h_first) { a = alpha_pass (a, P.h, ox); a = alpha_pass (a, P.v, oy); }
    else { a = alpha_pass (a, P.v, oy); a = alpha_pass (a, P.h, ox); }
    if (PLOUT) {
      store_planar_px (P, out, ox, oy, pack_px (a, r, g, b, P.sel));
      continue;
    }
    unsigned *dst = (unsigned *) (out + P.off_out + (size_t) oy * P.stride_out) + ox;
    *dst = pack_px (a, r, g, b, P.sel);
  }
}

}  // namespace b200
