// gstreamer_b200/csrc/vcs_planes_fast.cuh — word-wide kernel for the plane-scaling fast path (product code, sm_90a).
//
// Same arithmetic as vcs_planes_kernel's PM_SCALE branch (vcs_planes.cuh; gst_video_scaler_2d, video-scaler.c:1451-1640, on one
// plane of 1- or 2-byte pixels with video_scale_h_near_u8 / video_scale_h_2tap_1u8 / video_scale_h_ntap_u8 and
// video_scale_v_*_u8), horizontal pass first, organised like vcs_ntap_kernel (vcs_ntap.cuh) instead of one thread per byte:
//
//  A  the tile's source region is staged once with 32-bit loads: S4[group of 4 lines][component][word column] holds the
//     4 lines of one word column as one uint4 (interleaved UV pairs are split into two byte planes on the way in)
//  B  horizontal pass: a thread owns one output column x 4 consecutive source lines.  n-tap: one funnel shift brings the
//     window's bytes to a word boundary, IDP.4A.U8.S8 against 4 packed taps, (acc+32)>>6 saturated; 2-tap: the two source
//     bytes of the 4 lines are gathered into two words and lerped on 16-bit lanes ((a*(256-f) + b*f) >> 8, ldreslinb); copy:
//     a byte select.  The four lines leave as ONE word (transposed), so that
//  C  the vertical pass finds the lines of its window in consecutive bytes: funnel shift by the window's first line,
//     IDP.4A / lerp_v_u8 / byte select, one byte (or one U,V pair) stored per thread, lanes on consecutive columns.
//
// vcs_planes_kernel runs far below the HBM roofline on a 4K -> 1080p NV12 frame: four
// output rows per CTA made it filter every source line 3.5 times, byte by byte from global memory.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "common.h"
#include "vcs_device.h"
#include "vcs_kernels.cuh"
#include "vcs_lanczos2.cuh"      // packed-byte helpers
#include "vcs_light.cuh"         // light_lerp
#include "vcs_plan.h"

namespace b200 {

struct PlaneFastDev {
  unsigned long long src_off, dst_off;
  int sstride, dstride, iw, ih, ow, oh;
  int tw, th, rows, pitch;       // tile (output pixels x rows), staged source lines (multiple of 4), word columns per staged line
  int ntw_h, ntw_v;              // packed tap words per output column / row (n-tap axes)
  int hspan, vspan;
  unsigned swz;                  // 4-byte pixels: output byte c takes component (swz >> 4c) & 3; 0 = same order
  const uint32_t *hoff, *voff;   // first source pixel / line of each output column / row
  const int16_t *hcoef, *vcoef;  // 2-tap axes: the fraction / the weight of the second line
  const int *h_packed, *v_packed;
};

constexpr int PLF_THREADS = 256;

// CompStore form of a plane kernel's store: NC bytes of output pixel byte column xb, row y of the launch's plane k, item i
// (base = the destination plane's first byte)
template <int NC> __device__ __forceinline__ void comp_store (const CompStore & S, int k, int i, uint8_t *base, int stride,
    int xb, int y, const int (&v)[NC])
{
  const int X = S.px[k][i] + xb, Y = S.py[k][i] + y;
  if (X < 0 || X + NC > S.dw[k] || Y < 0 || Y >= S.dh[k]) return;
  uint8_t *p = base + (size_t) Y * stride + X;
  const int a = S.alpha[i];
#pragma unroll
  for (int c = 0; c < NC; c++) p[c] = (uint8_t) (a >= 256 ? v[c] : (p[c] * (256 - a) + v[c] * a) >> 8);
}

// the NC words of one pixel column (one per component) as a single shared-memory access
template <int NC> __device__ __forceinline__ void plf_ld (const unsigned *p, unsigned (&v)[NC])
{
  if (NC == 4) { const uint4 q = *(const uint4 *) p; v[0] = q.x; v[1 % NC] = q.y; v[2 % NC] = q.z; v[3 % NC] = q.w; }
  else if (NC == 2) { const uint2 q = *(const uint2 *) p; v[0] = q.x; v[1 % NC] = q.y; }
  else v[0] = p[0];
}
template <int NC> __device__ __forceinline__ void plf_st (unsigned *p, const unsigned (&v)[NC])
{
  if (NC == 4) *(uint4 *) p = make_uint4 (v[0], v[1 % NC], v[2 % NC], v[3 % NC]);
  else if (NC == 2) *(uint2 *) p = make_uint2 (v[0], v[1 % NC]);
  else p[0] = v[0];
}

// HM / VM: PassMode of the axis (1 copy / nearest, 2 two taps, 3 n taps); NC: bytes per pixel (1, 2 for interleaved UV, 4 for
// packed RGB); NTW > 0: every n-tap axis uses exactly NTW packed tap words (straight-line FIRs), 0: run-time loops
template <int HM, int VM, int NC, int NTW, class ST>
__device__ __forceinline__ void planes_fast_body (const PlaneFastDev & Q, const VcsBatch & frames, const ST & S)
{
  extern __shared__ __align__ (16) unsigned plsm[];
  const int ngr = Q.rows / 4, groups = ngr + 1 + Q.ntw_v;
  uint4 *S4 = (uint4 *) plsm;                                    // [ngr][NC][pitch]
  unsigned *T = (unsigned *) (S4 + ngr * NC * Q.pitch + 2);      // [groups][tw][NC]: 4 h-scaled lines per word
  int *TH = (int *) (T + groups * Q.tw * NC);                    // [tw][ntw_h] packed taps, or [tw] fractions
  int *TV = TH + Q.tw * max (Q.ntw_h, 1);                        // [th][ntw_v] packed taps, or [th] weights
  unsigned *vrow = (unsigned *) (TV + Q.th * max (Q.ntw_v, 1));  // [th] first source line of each output row
  const int tid = threadIdx.x;
  const uint8_t *__restrict__ src = frames.in[blockIdx.z] + Q.src_off;
  uint8_t *__restrict__ dst = frames.out[blockIdx.z] + Q.dst_off;

  const int ox0 = blockIdx.x * Q.tw, oy0 = blockIdx.y * Q.th;
  const int tw = min (Q.tw, Q.ow - ox0), th = min (Q.th, Q.oh - oy0);
  const int cx0 = (int) Q.hoff[ox0], cx1 = (int) Q.hoff[ox0 + tw - 1] + Q.hspan;
  const int ry0 = (int) Q.voff[oy0], ry1 = (int) Q.voff[oy0 + th - 1] + Q.vspan;
  const int cxa = cx0 & ~3, R = ry1 - ry0, ng = (cx1 - cxa + 3) >> 2;

  if (HM == 3)
    for (int i = tid; i < tw * Q.ntw_h; i += PLF_THREADS) TH[i] = __ldg (Q.h_packed + (size_t) ox0 * Q.ntw_h + i);
  else if (HM == 2 && tid < tw) TH[tid] = (int) Q.hcoef[ox0 + tid];
  if (VM == 3)
    for (int i = tid; i < th * Q.ntw_v; i += PLF_THREADS) TV[i] = __ldg (Q.v_packed + (size_t) oy0 * Q.ntw_v + i);
  else if (VM == 2 && tid < th) TV[tid] = (int) Q.vcoef[oy0 + tid];
  if (tid < th) vrow[tid] = Q.voff[oy0 + tid] - (unsigned) ry0;

  // ---------------------------------------------------------------- A: stage the source region
  // Lines past the plane's last one repeat it and words past the line's last whole word repeat that word: neither is ever
  // met by a non-zero tap (the reference folds its edge taps inward, the 2-tap fraction is 0 at the edge), they only have
  // to be readable.
  const int RG = (R + 3) >> 2;
  const int last_word = Q.sstride - 4;                            // byte offset of the last whole word of a line
  for (int i = tid; i < RG * ng; i += PLF_THREADS) {
    const int g = i / ng, j = i - g * ng;
    unsigned w[NC][4];
#pragma unroll
    for (int l = 0; l < 4; l++) {
      const uint8_t *line = src + (size_t) min (ry0 + 4 * g + l, Q.ih - 1) * Q.sstride;
      if (NC == 1) {
        w[0][l] = __ldg ((const unsigned *) (line + min (cxa + 4 * j, last_word)));
      } else if (NC == 2) {
        const unsigned a = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 2, last_word)));
        const unsigned b = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 2 + 4, last_word)));
        w[0][l] = __byte_perm (a, b, 0x6420);
        w[1 % NC][l] = __byte_perm (a, b, 0x7531);
      } else {                                                     // 4-byte pixels: 4 pixels -> one word per component
        const unsigned p0 = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 4, last_word)));
        const unsigned p1 = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 4 + 4, last_word)));
        const unsigned p2 = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 4 + 8, last_word)));
        const unsigned p3 = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 4 + 12, last_word)));
        const unsigned a01 = __byte_perm (p0, p1, 0x5140), a23 = __byte_perm (p2, p3, 0x5140);   // c0 c0' c1 c1' of pixels (0,1) / (2,3)
        const unsigned b01 = __byte_perm (p0, p1, 0x7362), b23 = __byte_perm (p2, p3, 0x7362);   // c2 c2' c3 c3'
        w[0][l] = __byte_perm (a01, a23, 0x5410); w[1 % NC][l] = __byte_perm (a01, a23, 0x7632);
        w[2 % NC][l] = __byte_perm (b01, b23, 0x5410); w[3 % NC][l] = __byte_perm (b01, b23, 0x7632);
      }
    }
#pragma unroll
    for (int c = 0; c < NC; c++) S4[(g * NC + c) * Q.pitch + j] = make_uint4 (w[c][0], w[c][1], w[c][2], w[c][3]);
  }
  __syncthreads ();

  // ---------------------------------------------------------------- B: horizontal pass
  const int tx = tid % Q.tw, ph = tid / Q.tw, nph = PLF_THREADS / Q.tw;   // tw is 32, 64 or 128
  if (tx < tw) {
    const int base = (int) Q.hoff[ox0 + tx] - cxa;
    const int wi = base >> 2, sh = (base & 3) * 8;
    for (int g = ph; g < RG; g += nph) {
      unsigned oc[NC];
#pragma unroll
      for (int c = 0; c < NC; c++) {
        const uint4 *sp = S4 + (g * NC + c) * Q.pitch + wi;
        unsigned o;
        if (HM == 3) {
          int acc[4] = {32, 32, 32, 32};
          uint4 lo = sp[0];
          const int *taps = TH + tx * Q.ntw_h;
#pragma unroll (NTW > 0 ? NTW : 2)
          for (int k = 0; k < (NTW > 0 ? NTW : Q.ntw_h); k++) {
            const int t = taps[k];
            const uint4 hi = sp[k + 1];
            acc[0] = dp4a_u8s8 (__funnelshift_r (lo.x, hi.x, sh), t, acc[0]);
            acc[1] = dp4a_u8s8 (__funnelshift_r (lo.y, hi.y, sh), t, acc[1]);
            acc[2] = dp4a_u8s8 (__funnelshift_r (lo.z, hi.z, sh), t, acc[2]);
            acc[3] = dp4a_u8s8 (__funnelshift_r (lo.w, hi.w, sh), t, acc[3]);
            lo = hi;
          }
          // (acc+32)>>6 saturated to u8 (video-orc.orc:2474-2481); the 4 lines of the column in one word
          o = pack_sat2 (acc[1] >> 6, acc[0] >> 6, pack_sat2 (acc[3] >> 6, acc[2] >> 6, 0u));
        } else if (HM == 2) {
          const uint4 lo = sp[0], hi = sp[1];
          const unsigned w0 = __funnelshift_r (lo.x, hi.x, sh), w1 = __funnelshift_r (lo.y, hi.y, sh);
          const unsigned w2 = __funnelshift_r (lo.z, hi.z, sh), w3 = __funnelshift_r (lo.w, hi.w, sh);
          const unsigned a = __byte_perm (__byte_perm (w0, w1, 0x0040), __byte_perm (w2, w3, 0x0040), 0x5410);
          const unsigned b = __byte_perm (__byte_perm (w0, w1, 0x0051), __byte_perm (w2, w3, 0x0051), 0x5410);
          const unsigned f = (unsigned) TH[tx];
          o = light_lerp (a, b, 256u - f, f, 0u);                 // (a*(256-f) + b*f) >> 8 on every byte (ldreslinb)
        } else {
          const unsigned s01 = (unsigned) (base & 3) | (unsigned) (4 + (base & 3)) << 4;
          const uint4 a = sp[0];
          o = __byte_perm (__byte_perm (a.x, a.y, s01), __byte_perm (a.z, a.w, s01), 0x5410);
        }
        oc[c] = o;
      }
      plf_st<NC> (T + (g * Q.tw + tx) * NC, oc);
    }
  }
  __syncthreads ();

  // ---------------------------------------------------------------- C: vertical pass, store
  if (tx < tw) {
    const int gs = Q.tw * NC;                                     // words between consecutive groups of one column
    uint8_t *dp = dst + (size_t) (oy0 + ph) * Q.dstride + (size_t) (ox0 + tx) * NC;
    const size_t dstep = (size_t) Q.dstride * nph;
    for (int ty = ph; ty < th; ty += nph, dp += dstep) {
      const int rb = (int) vrow[ty];
      const int sh = (rb & 3) * 8;
      int v[NC];
      const unsigned *tp = T + ((rb >> 2) * Q.tw + tx) * NC;
      unsigned lo[NC];
      plf_ld<NC> (tp, lo);
      if (VM == 3) {
        int acc[NC];
#pragma unroll
        for (int c = 0; c < NC; c++) acc[c] = 32;
        const int *taps = TV + ty * Q.ntw_v;
#pragma unroll (NTW > 0 ? NTW : 2)
        for (int k = 0; k < (NTW > 0 ? NTW : Q.ntw_v); k++) {
          unsigned hi[NC];
          plf_ld<NC> (tp + (k + 1) * gs, hi);
          const int t = taps[k];
#pragma unroll
          for (int c = 0; c < NC; c++) { acc[c] = dp4a_u8s8 (__funnelshift_r (lo[c], hi[c], sh), t, acc[c]); lo[c] = hi[c]; }
        }
#pragma unroll
        for (int c = 0; c < NC; c++) v[c] = min (max (acc[c] >> 6, 0), 255);
      } else if (VM == 2) {
        unsigned hi[NC];
        plf_ld<NC> (tp + gs, hi);
        const int wt = TV[ty];
#pragma unroll
        for (int c = 0; c < NC; c++) {
          const unsigned w = __funnelshift_r (lo[c], hi[c], sh);
          v[c] = lerp_v_u8 ((int) (w & 0xffu), (int) ((w >> 8) & 0xffu), wt);
        }
      } else {
#pragma unroll
        for (int c = 0; c < NC; c++) v[c] = (int) ((lo[c] >> sh) & 0xffu);
      }
      if constexpr (ST::fused) comp_store<NC> (S, 0, blockIdx.z, dst, Q.dstride, (ox0 + tx) * NC, oy0 + ty, v);
      else if (NC == 1) *dp = (uint8_t) v[0];
      else if (NC == 2) *(unsigned short *) dp = (unsigned short) ((unsigned) v[0] | ((unsigned) v[1 % NC] << 8));
      else {                                                       // 4-byte pixel, optionally in another byte order (PlaneFastDev::swz)
        const unsigned px = (unsigned) v[0] | ((unsigned) v[1 % NC] << 8) | ((unsigned) v[2 % NC] << 16) | ((unsigned) v[3 % NC] << 24);
        *(unsigned *) dp = Q.swz ? __byte_perm (px, 0, Q.swz) : px;
      }
    }
  }
}

template <int HM, int VM, int NC, int NTW = 0>
__global__ void __launch_bounds__ (PLF_THREADS, 2)
vcs_planes_fast_kernel (const PlaneFastDev Q, const VcsBatch frames)
{
  planes_fast_body<HM, VM, NC, NTW> (Q, frames, NoStore ());
}

// the CompStore form (b200_comp_blend_convert's fused route)
template <int HM, int VM, int NC, int NTW = 0>
__global__ void __launch_bounds__ (PLF_THREADS, 2)
vcs_planes_fast_comp_kernel (const PlaneFastDev Q, const VcsBatch frames, const CompStore S)
{
  planes_fast_body<HM, VM, NC, NTW> (Q, frames, S);
}

// ---- vertical pass first (gst_video_scaler_2d picks it whenever the plane shrinks vertically, video-scaler.c:1515-1520) -----------
//  A' the source region is staged TRANSPOSED: one word = the 4 lines (of a group) of ONE pixel column, a uint4 = 4 adjacent
//     columns (4 LDG.32, a 4 x 4 byte transpose in 8 PRMT, one STS.128; UV pairs split into two planes first)
//  B' vertical pass: a thread owns 4 adjacent columns of one output row: per 4 taps one LDS.128, 4 funnel shifts by the window's
//     first line, 4 IDP.4A; the four results leave as one word of 4 PIXELS in T[row][column word] - the natural layout for
//  C' the horizontal pass: a thread owns one output byte (or U,V pair): funnel shift to the window's first pixel, IDP.4A / lerp /
//     byte select on the v-scaled row, one store, lanes on consecutive columns.
// NTW > 0: every n-tap axis of the plane uses exactly NTW packed tap words (straight-line FIRs); 0: run-time loops
template <int HM, int VM, int NC, int NTW, class ST>
__device__ __forceinline__ void planes_fast_vfirst_body (const PlaneFastDev & Q, const VcsBatch & frames, const ST & S)
{
  extern __shared__ __align__ (16) unsigned plsm[];
  const int ngr = Q.rows / 4;
  uint4 *S4 = (uint4 *) plsm;                                    // [ngr + 1 + ntw_v][NC][pitch]: 4 columns x (4 lines per word)
  unsigned *T = (unsigned *) (S4 + (ngr + 1 + Q.ntw_v) * NC * Q.pitch + 2);   // [th][NC][pitch]: v-scaled rows, 4 pixels per word
  const int trow = Q.pitch;                                      // (pitch leaves room for the h window's ntw_h + 1 words past the last column)
  int *TH = (int *) (T + Q.th * NC * trow);
  int *TV = TH + Q.tw * max (Q.ntw_h, 1);
  unsigned *vrow = (unsigned *) (TV + Q.th * max (Q.ntw_v, 1));
  const int tid = threadIdx.x;
  const uint8_t *__restrict__ src = frames.in[blockIdx.z] + Q.src_off;
  uint8_t *__restrict__ dst = frames.out[blockIdx.z] + Q.dst_off;

  const int ox0 = blockIdx.x * Q.tw, oy0 = blockIdx.y * Q.th;
  const int tw = min (Q.tw, Q.ow - ox0), th = min (Q.th, Q.oh - oy0);
  const int cx0 = (int) Q.hoff[ox0], cx1 = (int) Q.hoff[ox0 + tw - 1] + Q.hspan;
  const int ry0 = (int) Q.voff[oy0], ry1 = (int) Q.voff[oy0 + th - 1] + Q.vspan;
  const int cxa = cx0 & ~3, R = ry1 - ry0, ng = (cx1 - cxa + 3) >> 2;

  if (HM == 3)
    for (int i = tid; i < tw * Q.ntw_h; i += PLF_THREADS) TH[i] = __ldg (Q.h_packed + (size_t) ox0 * Q.ntw_h + i);
  else if (HM == 2 && tid < tw) TH[tid] = (int) Q.hcoef[ox0 + tid];
  if (VM == 3)
    for (int i = tid; i < th * Q.ntw_v; i += PLF_THREADS) TV[i] = __ldg (Q.v_packed + (size_t) oy0 * Q.ntw_v + i);
  else if (VM == 2 && tid < th) TV[tid] = (int) Q.vcoef[oy0 + tid];
  if (tid < th) vrow[tid] = Q.voff[oy0 + tid] - (unsigned) ry0;

  // ---------------------------------------------------------------- A': stage, transposed
  const int RG = (R + 3) >> 2;
  const int last_word = Q.sstride - 4;
  const unsigned magic = 0xffffffffu / (unsigned) ng + 1u;       // i / ng by multiplication: exact for i, ng < 2^16 (a tile has a few thousand items)
  for (int i = tid; i < RG * ng; i += PLF_THREADS) {
    const int g = ng > 1 ? (int) __umulhi ((unsigned) i, magic) : i, j = i - g * ng;
    unsigned w[NC][4];
#pragma unroll
    for (int l = 0; l < 4; l++) {
      const uint8_t *line = src + (size_t) min (ry0 + 4 * g + l, Q.ih - 1) * Q.sstride;
      if (NC == 1) {
        w[0][l] = __ldg ((const unsigned *) (line + min (cxa + 4 * j, last_word)));
      } else if (NC == 2) {
        const unsigned a = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 2, last_word)));
        const unsigned b = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 2 + 4, last_word)));
        w[0][l] = __byte_perm (a, b, 0x6420);
        w[1 % NC][l] = __byte_perm (a, b, 0x7531);
      } else {                                                     // 4-byte pixels: 4 pixels -> one word per component
        const unsigned p0 = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 4, last_word)));
        const unsigned p1 = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 4 + 4, last_word)));
        const unsigned p2 = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 4 + 8, last_word)));
        const unsigned p3 = __ldg ((const unsigned *) (line + min ((cxa + 4 * j) * 4 + 12, last_word)));
        const unsigned a01 = __byte_perm (p0, p1, 0x5140), a23 = __byte_perm (p2, p3, 0x5140);   // c0 c0' c1 c1' of pixels (0,1) / (2,3)
        const unsigned b01 = __byte_perm (p0, p1, 0x7362), b23 = __byte_perm (p2, p3, 0x7362);   // c2 c2' c3 c3'
        w[0][l] = __byte_perm (a01, a23, 0x5410); w[1 % NC][l] = __byte_perm (a01, a23, 0x7632);
        w[2 % NC][l] = __byte_perm (b01, b23, 0x5410); w[3 % NC][l] = __byte_perm (b01, b23, 0x7632);
      }
    }
#pragma unroll
    for (int c = 0; c < NC; c++) {
      // 4 x 4 byte transpose: w[c][l] = pixels 0..3 of line l  ->  column k = lines 0..3 of pixel k
      const unsigned a01 = __byte_perm (w[c][0], w[c][1], 0x5140), a23 = __byte_perm (w[c][2], w[c][3], 0x5140);   // p0l0 p0l1 p1l0 p1l1
      const unsigned b01 = __byte_perm (w[c][0], w[c][1], 0x7362), b23 = __byte_perm (w[c][2], w[c][3], 0x7362);   // p2l0 p2l1 p3l0 p3l1
      S4[(g * NC + c) * Q.pitch + j] = make_uint4 (__byte_perm (a01, a23, 0x5410), __byte_perm (a01, a23, 0x7632),
          __byte_perm (b01, b23, 0x5410), __byte_perm (b01, b23, 0x7632));
    }
  }
  __syncthreads ();

  // ---------------------------------------------------------------- B': vertical pass
  for (int i = tid; i < th * ng; i += PLF_THREADS) {
    const int ty = ng > 1 ? (int) __umulhi ((unsigned) i, magic) : i, j = i - ty * ng;
    const int rb = (int) vrow[ty];
    const int sh = (rb & 3) * 8;
#pragma unroll
    for (int c = 0; c < NC; c++) {
      const uint4 *sp = S4 + ((rb >> 2) * NC + c) * Q.pitch + j;
      const int gstep = NC * Q.pitch;
      unsigned o;
      if (VM == 3) {
        int acc[4] = {32, 32, 32, 32};
        uint4 lo = sp[0];
        const int *taps = TV + ty * Q.ntw_v;
#pragma unroll
        for (int k = 0; k < (NTW > 0 ? NTW : Q.ntw_v); k++) {
          const int t = taps[k];
          const uint4 hi = sp[(k + 1) * gstep];
          acc[0] = dp4a_u8s8 (__funnelshift_r (lo.x, hi.x, sh), t, acc[0]);
          acc[1] = dp4a_u8s8 (__funnelshift_r (lo.y, hi.y, sh), t, acc[1]);
          acc[2] = dp4a_u8s8 (__funnelshift_r (lo.z, hi.z, sh), t, acc[2]);
          acc[3] = dp4a_u8s8 (__funnelshift_r (lo.w, hi.w, sh), t, acc[3]);
          lo = hi;
        }
        o = pack_sat2 (acc[1] >> 6, acc[0] >> 6, pack_sat2 (acc[3] >> 6, acc[2] >> 6, 0u));
      } else if (VM == 2) {
        const uint4 lo = sp[0], hi = sp[gstep];
        const unsigned w0 = __funnelshift_r (lo.x, hi.x, sh), w1 = __funnelshift_r (lo.y, hi.y, sh);
        const unsigned w2 = __funnelshift_r (lo.z, hi.z, sh), w3 = __funnelshift_r (lo.w, hi.w, sh);
        const unsigned a = __byte_perm (__byte_perm (w0, w1, 0x0040), __byte_perm (w2, w3, 0x0040), 0x5410);
        const unsigned b = __byte_perm (__byte_perm (w0, w1, 0x0051), __byte_perm (w2, w3, 0x0051), 0x5410);
        const unsigned p = (unsigned) TV[ty];
        // bits 8..15 of s0*(256-p) + s1*p + 128 == the wrapping 16-bit s0 + (((s1-s0)*p + 128) >> 8) of the reference (vcs_light.cuh)
        o = light_lerp (a, b, 256u - p, p, 0x00800080u);
      } else {
        const unsigned s01 = (unsigned) (rb & 3) | (unsigned) (4 + (rb & 3)) << 4;
        const uint4 a = sp[0];
        o = __byte_perm (__byte_perm (a.x, a.y, s01), __byte_perm (a.z, a.w, s01), 0x5410);
      }
      T[(ty * NC + c) * trow + j] = o;
    }
  }
  __syncthreads ();

  // ---------------------------------------------------------------- C': horizontal pass, store
  const int tx = tid % Q.tw, ph = tid / Q.tw, nph = PLF_THREADS / Q.tw;
  if (tx < tw) {
    const int base = (int) Q.hoff[ox0 + tx] - cxa;
    const int wi = base >> 2, sh = (base & 3) * 8;
    uint8_t *dp = dst + (size_t) (oy0 + ph) * Q.dstride + (size_t) (ox0 + tx) * NC;
    const size_t dstep = (size_t) Q.dstride * nph;
    for (int ty = ph; ty < th; ty += nph, dp += dstep) {
      int v[NC];
#pragma unroll
      for (int c = 0; c < NC; c++) {
        const unsigned *tp = T + (ty * NC + c) * trow + wi;
        if (HM == 3) {
          int acc = 32;
          unsigned lo = tp[0];
          const int *taps = TH + tx * Q.ntw_h;
#pragma unroll
          for (int k = 0; k < (NTW > 0 ? NTW : Q.ntw_h); k++) {
            const unsigned hi = tp[k + 1];
            acc = dp4a_u8s8 (__funnelshift_r (lo, hi, sh), taps[k], acc);
            lo = hi;
          }
          v[c] = min (max (acc >> 6, 0), 255);
        } else if (HM == 2) {
          const unsigned w = __funnelshift_r (tp[0], tp[1], sh);
          v[c] = lerp_h_u8 ((int) (w & 0xffu), (int) ((w >> 8) & 0xffu), TH[tx]);
        } else {
          v[c] = (int) ((tp[0] >> sh) & 0xffu);
        }
      }
      if constexpr (ST::fused) comp_store<NC> (S, 0, blockIdx.z, dst, Q.dstride, (ox0 + tx) * NC, oy0 + ty, v);
      else if (NC == 1) *dp = (uint8_t) v[0];
      else if (NC == 2) *(unsigned short *) dp = (unsigned short) ((unsigned) v[0] | ((unsigned) v[1 % NC] << 8));
      else {                                                       // 4-byte pixel, optionally in another byte order (PlaneFastDev::swz)
        const unsigned px = (unsigned) v[0] | ((unsigned) v[1 % NC] << 8) | ((unsigned) v[2 % NC] << 16) | ((unsigned) v[3 % NC] << 24);
        *(unsigned *) dp = Q.swz ? __byte_perm (px, 0, Q.swz) : px;
      }
    }
  }
}

template <int HM, int VM, int NC, int NTW = 0>
__global__ void __launch_bounds__ (PLF_THREADS, 2)
vcs_planes_fast_vfirst_kernel (const PlaneFastDev Q, const VcsBatch frames)
{
  planes_fast_vfirst_body<HM, VM, NC, NTW> (Q, frames, NoStore ());
}

// the CompStore form (b200_comp_blend_convert's fused route)
template <int HM, int VM, int NC, int NTW = 0>
__global__ void __launch_bounds__ (PLF_THREADS, 2)
vcs_planes_fast_vfirst_comp_kernel (const PlaneFastDev Q, const VcsBatch frames, const CompStore S)
{
  planes_fast_vfirst_body<HM, VM, NC, NTW> (Q, frames, S);
}

// ------------------------------------------------------------------------------------ host side
struct PlaneFastState {
  bool ok = false;
  PlaneFastDev dev;
  int hm = 0, vm = 0, nc = 0;
  bool vfirst = false;
  int ntw = 0;                   // the n-tap axes' common tap-word count (0: they differ, run-time loops)
  size_t smem = 0;
  uint32_t *d_hoff = nullptr, *d_voff = nullptr;
  int16_t *d_hcoef = nullptr, *d_vcoef = nullptr;
  int *d_hp = nullptr, *d_vp = nullptr;
};

template <class ST> struct PlaneFastFn { using type = void (*) (const PlaneFastDev, const VcsBatch, const CompStore); };
template <> struct PlaneFastFn<NoStore> { using type = void (*) (const PlaneFastDev, const VcsBatch); };
template <class ST = NoStore> using plane_fast_fn = typename PlaneFastFn<ST>::type;

// the kernel of a store form: vcs_planes_fast[_vfirst]_kernel, or its CompStore form
template <class ST, bool VFIRST, int H, int V, int NC, int NTW> constexpr plane_fast_fn<ST> plf_kernel ()
{
  if constexpr (ST::fused && VFIRST) return vcs_planes_fast_vfirst_comp_kernel<H, V, NC, NTW>;
  else if constexpr (ST::fused) return vcs_planes_fast_comp_kernel<H, V, NC, NTW>;
  else if constexpr (VFIRST) return vcs_planes_fast_vfirst_kernel<H, V, NC, NTW>;
  else return vcs_planes_fast_kernel<H, V, NC, NTW>;
}

// the instantiation a plane runs; the CompStore forms exist for the 1- and 2-byte pixels of 4:2:0 planes only
template <class ST = NoStore>
inline plane_fast_fn<ST> plane_fast_kernel_for (int hm, int vm, int nc, bool vfirst, int ntw = 0)
{
#define PLF_PICK(H, V)                                                                         \
  if (hm == H && vm == V) {                                                                    \
    if constexpr (!ST::fused) {                                                                \
      if (nc == 4 && vfirst && ntw == 2 && (H == 3 || V == 3)) return vcs_planes_fast_vfirst_kernel<H, V, 4, 2>;   \
      if (nc == 4 && !vfirst && ntw == 2 && (H == 3 || V == 3)) return vcs_planes_fast_kernel<H, V, 4, 2>;   \
      if (nc == 4 && !vfirst && ntw == 1 && (H == 3 || V == 3)) return vcs_planes_fast_kernel<H, V, 4, 1>;   \
      if (nc == 4) return vfirst ? vcs_planes_fast_vfirst_kernel<H, V, 4> : vcs_planes_fast_kernel<H, V, 4>;   \
    }                                                                                          \
    if (nc == 4) return nullptr;                                                               \
    if (!vfirst && ntw == 1 && (H == 3 || V == 3)) return nc == 1 ? plf_kernel<ST, false, H, V, 1, 1> () : plf_kernel<ST, false, H, V, 2, 1> ();   \
    if (vfirst && ntw == 2 && (H == 3 || V == 3)) return nc == 1 ? plf_kernel<ST, true, H, V, 1, 2> () : plf_kernel<ST, true, H, V, 2, 2> ();   \
    if (vfirst && ntw == 1 && (H == 3 || V == 3)) return nc == 1 ? plf_kernel<ST, true, H, V, 1, 1> () : plf_kernel<ST, true, H, V, 2, 1> ();   \
    if (vfirst) return nc == 1 ? plf_kernel<ST, true, H, V, 1, 0> () : plf_kernel<ST, true, H, V, 2, 0> ();   \
    return nc == 1 ? plf_kernel<ST, false, H, V, 1, 0> () : plf_kernel<ST, false, H, V, 2, 0> ();       \
  }
  PLF_PICK (1, 1) PLF_PICK (1, 2) PLF_PICK (1, 3) PLF_PICK (2, 1) PLF_PICK (2, 2) PLF_PICK (2, 3)
  PLF_PICK (3, 1) PLF_PICK (3, 2) PLF_PICK (3, 3)
#undef PLF_PICK
  return nullptr;
}

// geometry + eligibility of one PM_SCALE plane; false leaves the plane to vcs_planes_kernel
inline bool plan_plane_fast (const PlanePlan & q, int sstride, unsigned long long src_off, int dstride, unsigned long long dst_off,
    PlaneFastState * st, std::vector<int32_t> * hp, std::vector<int32_t> * vp)
{
  st->ok = false;
  if (q.mode != PM_SCALE || (q.ne != 1 && q.ne != 2 && q.ne != 4) || (q.swz && q.ne != 4)) return false;
  if ((sstride & 3) || (src_off & 3) || sstride < 4) return false;
  if (q.ne == 2 && ((dstride & 1) || (dst_off & 1))) return false;
  if (q.ne == 4 && ((dstride & 3) || (dst_off & 3))) return false;
  const AxisPlan & H = q.h, & V = q.v;
  if (H.mode < 1 || H.mode > 3 || V.mode < 1 || V.mode > 3) return false;
  int ntw_h = 0, ntw_v = 0;
  if (!pack_taps_s8 (H, &ntw_h, hp) || !pack_taps_s8 (V, &ntw_v, vp)) return false;
  if (H.mode == PASS_2TAP) for (int16_t f : H.coef) if (f < 0 || f > 255) return false;     // 8-bit fractions (ldreslinb)
  if (V.mode == PASS_2TAP && !q.h_first) for (int16_t w : V.coef) if (w < 0 || w > 256) return false;   // lane form of lerp_v_u8
  static const int shapes[][2] = {{128, 64}, {128, 32}, {128, 16}, {64, 32}, {128, 8}, {64, 16}, {32, 32}, {64, 8}, {32, 16},
                                  {64, 4}, {32, 8}, {32, 4}};
  auto smem = [&] (TileShape & t) -> size_t {
    const int ngr = t.rows / 4, groups = ngr + 1 + ntw_v;
    t.pitch = t.cols / 4 + 2 + std::max (ntw_h, 1);
    return ((q.h_first ? ((size_t) ngr * q.ne * t.pitch + 2) * 4 + (size_t) groups * t.tw * q.ne
                       : ((size_t) groups * q.ne * t.pitch + 2) * 4 + (size_t) t.th * q.ne * t.pitch) +
        (size_t) t.tw * std::max (ntw_h, 1) + (size_t) t.th * std::max (ntw_v, 1) + t.th + 8) * 4;
  };
  TileShape s;
  if (!search_tile_shape (H, V, shapes, (int) std::size (shapes), "B200_PLF_SHAPE", smem, &s)) return false;
  PlaneFastDev & d = st->dev;
  d.tw = s.tw; d.th = s.th; d.rows = s.rows; d.pitch = s.pitch; st->smem = s.smem;
  d.src_off = src_off; d.dst_off = dst_off; d.sstride = sstride; d.dstride = dstride;
  d.iw = q.iw; d.ih = q.ih; d.ow = q.ow; d.oh = q.oh;
  d.ntw_h = ntw_h; d.ntw_v = ntw_v; d.hspan = H.span; d.vspan = V.span; d.swz = q.swz;
  st->hm = H.mode; st->vm = V.mode; st->nc = q.ne; st->vfirst = !q.h_first;
  st->ntw = common_tap_words (H.mode, V.mode, ntw_h, ntw_v);
  st->ok = true;
  return true;
}

inline int prepare_plane_fast (const PlanePlan & q, const std::vector<int32_t> & hp, const std::vector<int32_t> & vp, PlaneFastState * st)
{
  int s;
  if ((s = upload (&st->d_hoff, q.h.offset.data (), q.h.offset.size ())) != B200_OK) return s;
  if ((s = upload (&st->d_voff, q.v.offset.data (), q.v.offset.size ())) != B200_OK) return s;
  if ((s = upload (&st->d_hcoef, q.h.coef.data (), q.h.coef.size ())) != B200_OK) return s;
  if ((s = upload (&st->d_vcoef, q.v.coef.data (), q.v.coef.size ())) != B200_OK) return s;
  if ((s = upload (&st->d_hp, hp.data (), hp.size ())) != B200_OK) return s;
  if ((s = upload (&st->d_vp, vp.data (), vp.size ())) != B200_OK) return s;
  st->dev.hoff = st->d_hoff; st->dev.voff = st->d_voff; st->dev.hcoef = st->d_hcoef; st->dev.vcoef = st->d_vcoef;
  st->dev.h_packed = st->d_hp; st->dev.v_packed = st->d_vp;
  if (st->nc != 4 && (s = allow_max_dyn_smem (plane_fast_kernel_for<CompStore> (st->hm, st->vm, st->nc, st->vfirst, st->ntw))) != B200_OK)
    return s;
  return allow_max_dyn_smem (plane_fast_kernel_for (st->hm, st->vm, st->nc, st->vfirst, st->ntw));
}

inline void free_plane_fast (PlaneFastState * st)
{
  cudaFree (st->d_hoff); cudaFree (st->d_voff); cudaFree (st->d_hcoef); cudaFree (st->d_vcoef); cudaFree (st->d_hp); cudaFree (st->d_vp);
}

template <class ST = NoStore>
inline int launch_plane_fast (const PlaneFastState & st, const VcsBatch & batch, int n, cudaStream_t stream, const ST & S = ST ())
{
  plane_fast_fn<ST> fn = plane_fast_kernel_for<ST> (st.hm, st.vm, st.nc, st.vfirst, st.ntw);
  if (!fn) return B200_ERR_STATE;
  const dim3 grid ((st.dev.ow + st.dev.tw - 1) / st.dev.tw, (st.dev.oh + st.dev.th - 1) / st.dev.th, n);
  if constexpr (ST::fused) fn <<<grid, PLF_THREADS, st.smem, stream>>> (st.dev, batch, S);
  else fn <<<grid, PLF_THREADS, st.smem, stream>>> (st.dev, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
