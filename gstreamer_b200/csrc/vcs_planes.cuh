// gstreamer_b200/csrc/vcs_planes.cuh — YUV -> same YUV family (NV12->NV12, NV21->NV21, I420/YV12 ->
// I420/YV12) and packed RGB -> the same packed RGB (one plane of 4-byte pixels, opt-in): the reference's
// plane-scaling fast path (product code, sm_90a); and the de-interleave of packed RGB -> RGBP / BGRP.
//
//   convert_scale_planes            gst-libs/gst/video/video-converter.c:7757-7769
//   setup_scale                     :7958-8245  (which kernel each plane gets; built on the host, vcs_plan.cpp)
//   convert_plane_{h,v,hv}_halve    :7399-7680  -> video_orc_planar_chroma_444_422 / _422_420 / _444_420
//   convert_plane_{h,v,hv}_double   :7348-7615  -> replication
//   gst_video_scaler_2d             gst-libs/gst/video/video-scaler.c:1451-1640 with video_scale_h_near_u8/_u16,
//                                   video_scale_h_2tap_1u8 (ldreslinb), video_scale_h_ntap_u8, video_scale_v_*_u8
//
// One thread per output byte; a CTA owns a 64 x 4 byte tile and stages the FIRST pass of its tile in shared memory
// (each intermediate byte computed once, rounded to 8 bits exactly where the reference rounds), the second pass
// reads it.  Windows too large for the stage fall back to direct evaluation.  One launch covers all planes of all
// frames of a batch.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"
#include "vcs_device.h"
#include "vcs_kernels.cuh"
#include "vcs_lanczos2.cuh"      // packed-byte averages
#include "vcs_plan.h"
#include "vcs_planes_fast.cuh"   // the word-wide kernel most PM_SCALE planes take

namespace b200 {

struct PlaneAxisDev {
  const uint32_t *offset;
  const int16_t *coef;
  int mode, n_taps;              // PassMode; taps per output
};

struct PlaneDev {
  unsigned long long src_off, dst_off;
  int sstride, dstride, iw, ih, ow, oh, ne, mode, h_first;
  int vec4;                      // copy / halve plane whose rows are word (source: double-word for h halving) aligned
  unsigned swz;                  // 4-byte pixels only: output byte c takes source byte (swz >> 4c) & 3; 0 = same order
  PlaneAxisDev h, v;
};

struct PlanesParams {
  PlaneDev pl[3];
  int n_planes;
};

// one pixel component of one line through the horizontal scaler
__device__ __forceinline__ int plane_h (const PlaneDev & Q, const uint8_t *line, int x, int c)
{
  const PlaneAxisDev & A = Q.h;
  if (A.mode == PASS_COPY) return line[(int) A.offset[x] * Q.ne + c];
  if (A.mode == PASS_2TAP) {                                       // ldreslinb; the second tap is unused (f == 0) at the edge
    const int i0 = (int) A.offset[x], f = A.coef[x];
    const int i1 = min (i0 + 1, Q.iw - 1);
    return lerp_h_u8 (line[i0 * Q.ne + c], line[i1 * Q.ne + c], f);
  }
  const int16_t *t = A.coef + (size_t) x * A.n_taps;
  const uint8_t *s = line + (int) A.offset[x] * Q.ne + c;
  int acc = 0;
  for (int k = 0; k < A.n_taps; k++) acc += (int) s[k * Q.ne] * (int) t[k];
  return fir_round_u8 (acc);
}

constexpr int PL_TW = 64, PL_TH = 4;          // output bytes x rows per CTA
constexpr int PL_STAGE_COLS = 1024;           // staged first-pass bytes per row (vertical first)
constexpr int PL_STAGE_ROWS = 40;             // staged first-pass rows (horizontal first)

__global__ void __launch_bounds__ (256)
vcs_planes_kernel (const PlanesParams P, const VcsBatch frames)
{
  // first-pass results of this CTA's tile, each computed once:
  //   vertical first:   stage[row of the tile][source byte column]   (4 x PL_STAGE_COLS)
  //   horizontal first: stage[source line][output byte of the tile]  (PL_STAGE_ROWS x 64)
  __shared__ uint8_t stage[PL_TH * PL_STAGE_COLS];
  const int plane = blockIdx.z % P.n_planes, frame = blockIdx.z / P.n_planes;
  const PlaneDev & Q = P.pl[plane];
  const int wbytes = Q.ow * Q.ne;
  const int xb0 = blockIdx.x * PL_TW, y0 = blockIdx.y * PL_TH;
  if (Q.mode != PM_SCALE && Q.mode != PM_DOUBLE && Q.vec4) {
    const uint8_t *__restrict__ src = frames.in[frame] + Q.src_off;
    uint8_t *__restrict__ dst = frames.out[frame] + Q.dst_off;
    // copy / halve planes with word-aligned rows: 4 output bytes per thread, the grid taken as a linear range of words
    const int wpr = wbytes >> 2;                                    // words per output row
    const long long wi = ((long long) blockIdx.y * gridDim.x + blockIdx.x) * 256 + threadIdx.x;
    const int wy = (int) (wi / wpr), wx = (int) (wi - (long long) wy * wpr);
    if (wy >= Q.oh) return;
    unsigned o;
    if (Q.mode == PM_COPY) {
      o = __ldg ((const unsigned *) (src + (size_t) wy * Q.sstride) + wx);
      if (Q.swz) o = __byte_perm (o, 0, Q.swz);                     // another byte order of the same 4-byte pixel
    } else if (Q.mode == PM_HALVE_V) {
      o = avg_ceil4 (__ldg ((const unsigned *) (src + (size_t) (2 * wy) * Q.sstride) + wx),
          __ldg ((const unsigned *) (src + (size_t) (2 * wy + 1) * Q.sstride) + wx));
    } else if (Q.mode == PM_HALVE_H) {
      const uint2 a = __ldg ((const uint2 *) (src + (size_t) wy * Q.sstride) + wx);
      o = avg_ceil4 (__byte_perm (a.x, a.y, 0x6420), __byte_perm (a.x, a.y, 0x7531));
    } else {                                                       // PM_HALVE_HV: lines first, then the byte pairs
      const uint2 a = __ldg ((const uint2 *) (src + (size_t) (2 * wy) * Q.sstride) + wx);
      const uint2 b = __ldg ((const uint2 *) (src + (size_t) (2 * wy + 1) * Q.sstride) + wx);
      const unsigned t = avg_ceil4 (a.x, b.x), u = avg_ceil4 (a.y, b.y);
      o = avg_ceil4 (__byte_perm (t, u, 0x6420), __byte_perm (t, u, 0x7531));
    }
    *((unsigned *) (dst + (size_t) wy * Q.dstride) + wx) = o;
    return;
  }
  if (xb0 >= wbytes || y0 >= Q.oh) return;                         // whole CTA outside this plane
  const int tx = threadIdx.x & (PL_TW - 1), ty = threadIdx.x >> 6;
  const int xb = xb0 + tx, y = y0 + ty;
  const bool live = xb < wbytes && y < Q.oh;
  const uint8_t *__restrict__ src = frames.in[frame] + Q.src_off;
  uint8_t *__restrict__ dst = frames.out[frame] + Q.dst_off;
  const int nes = Q.ne >> 1;                                        // ne is 1, 2 or 4 (shift 0, 1, 2): divide by shifting
  const int x = min (xb, wbytes - 1) >> nes, c = min (xb, wbytes - 1) - (x << nes);
  const int cs = Q.swz ? (int) ((Q.swz >> (4 * c)) & 3) : c;        // source component feeding output component c
  int v = 0;
  if (Q.mode != PM_SCALE) {
    if (!live) return;
    switch (Q.mode) {
      case PM_COPY:
        v = src[(size_t) y * Q.sstride + (x << nes) + cs];
        break;
      case PM_HALVE_V:                                             // avgub of the two lines
        v = (src[(size_t) (2 * y) * Q.sstride + xb] + src[(size_t) (2 * y + 1) * Q.sstride + xb] + 1) >> 1;
        break;
      case PM_HALVE_H:
        v = (src[(size_t) y * Q.sstride + 2 * xb] + src[(size_t) y * Q.sstride + 2 * xb + 1] + 1) >> 1;
        break;
      case PM_HALVE_HV: {                                          // vertical averages first, then the pair
        const uint8_t *a = src + (size_t) (2 * y) * Q.sstride + 2 * xb, *b = a + Q.sstride;
        const int t1 = (a[0] + b[0] + 1) >> 1, t2 = (a[1] + b[1] + 1) >> 1;
        v = (t1 + t2 + 1) >> 1;
        break;
      }
      default:                                                     // PM_DOUBLE
        v = src[(size_t) (Q.ih == Q.oh ? y : y >> 1) * Q.sstride + (Q.iw == Q.ow ? xb : xb >> 1)];
        break;
    }
    dst[(size_t) y * Q.dstride + xb] = (uint8_t) v;
    return;
  }

  const PlaneAxisDev & V = Q.v, & H = Q.h;
  const int rows = min (PL_TH, Q.oh - y0);
  const int xl = min (xb0 + PL_TW, wbytes) - 1;                     // last output byte of the tile
  const int px0 = xb0 >> nes, px1 = xl >> nes;                      // first / last output pixel
  const int hspan = H.mode == PASS_NTAP ? H.n_taps : (H.mode == PASS_2TAP ? 2 : 1);
  const int vspan = V.mode == PASS_NTAP ? V.n_taps : (V.mode == PASS_2TAP ? 2 : 1);
  auto vfilter = [&] (const uint8_t *s, int oy) -> int {            // s: first source line of output row oy, one byte column
    if (V.mode == PASS_COPY) return s[0];
    if (V.mode == PASS_2TAP) return lerp_v_u8 (s[0], s[Q.sstride], V.coef[oy]);
    const int16_t *t = V.coef + (size_t) oy * V.n_taps;
    int acc = 0;
    for (int k = 0; k < V.n_taps; k++) acc += (int) s[(size_t) k * Q.sstride] * (int) t[k];
    return fir_round_u8 (acc);
  };
  if (!Q.h_first) {
    // ---- vertical first: v-scale the source columns the tile's horizontal windows touch, once
    const int c0 = (int) H.offset[px0], c1 = min ((int) H.offset[px1] + hspan, Q.iw);     // source pixels [c0, c1)
    const int nb = (c1 - c0) * Q.ne;
    const bool staged = nb <= PL_STAGE_COLS;
    if (staged) {
      for (int i = threadIdx.x; i < rows * nb; i += 256) {
        const int r = (i >= nb) + (i >= 2 * nb) + (i >= 3 * nb), col = i - r * nb;      // rows <= 4: no division
        stage[r * PL_STAGE_COLS + col] = (uint8_t) vfilter (src + (size_t) V.offset[y0 + r] * Q.sstride + c0 * Q.ne + col, y0 + r);
      }
    }
    __syncthreads ();
    if (!live) return;
    auto vcol = [&] (int col) -> int {                             // v-scaled byte of source pixel `col`, component c
      if (staged) return stage[ty * PL_STAGE_COLS + (col - c0) * Q.ne + cs];
      return vfilter (src + (size_t) V.offset[y] * Q.sstride + col * Q.ne + cs, y);
    };
    const int i0 = (int) H.offset[x];
    if (H.mode == PASS_COPY) v = vcol (i0);
    else if (H.mode == PASS_2TAP) v = lerp_h_u8 (vcol (i0), vcol (min (i0 + 1, Q.iw - 1)), H.coef[x]);
    else {
      const int16_t *t = H.coef + (size_t) x * H.n_taps;
      int acc = 0;
      for (int k = 0; k < H.n_taps; k++) acc += vcol (i0 + k) * (int) t[k];
      v = fir_round_u8 (acc);
    }
  } else {
    // ---- horizontal first: h-scale the source lines the tile's vertical windows touch, once
    const int r0 = (int) V.offset[y0], r1 = min ((int) V.offset[y0 + rows - 1] + vspan, Q.ih);   // source lines [r0, r1)
    const int nr = r1 - r0, tw = xl - xb0 + 1;
    const bool staged = nr <= PL_STAGE_ROWS;
    if (staged) {
      // thread (tx, ty) fills column tx of source lines ty, ty + 4, ...
      if (tx < tw)
        for (int r = ty; r < nr; r += PL_TH)
          stage[r * PL_TW + tx] = (uint8_t) plane_h (Q, src + (size_t) (r0 + r) * Q.sstride, x, cs);
    }
    __syncthreads ();
    if (!live) return;
    auto hline = [&] (int line) -> int {                           // h-scaled byte of source line `line` at this thread's column
      if (staged) return stage[(line - r0) * PL_TW + tx];
      return plane_h (Q, src + (size_t) line * Q.sstride, x, cs);
    };
    const int l0 = (int) V.offset[y];
    if (V.mode == PASS_COPY) v = hline (l0);
    else if (V.mode == PASS_2TAP) v = lerp_v_u8 (hline (l0), hline (l0 + 1), V.coef[y]);
    else {
      const int16_t *t = V.coef + (size_t) y * V.n_taps;
      int acc = 0;
      for (int k = 0; k < V.n_taps; k++) acc += hline (l0 + k) * (int) t[k];
      v = fir_round_u8 (acc);
    }
  }
  dst[(size_t) y * Q.dstride + xb] = (uint8_t) v;
}

// copy / halve planes with word-aligned rows on their own: one thread = one output word, the grid exactly the plane's words
// (inside vcs_planes_kernel these modes ran on the byte kernel's grid with its register footprint, far below the HBM
// bandwidth).  Same arithmetic as the vec4 branch above (video_orc_planar_chroma_*, avgub).
__global__ void __launch_bounds__ (256)
vcs_planes_vec_kernel (const PlaneDev Q, const VcsBatch frames)
{
  const int wpr = (Q.ow * Q.ne) >> 2;                              // words per output row
  const int wx = blockIdx.x * 64 + (threadIdx.x & 63), wy = blockIdx.y * 4 + (threadIdx.x >> 6);
  if (wx >= wpr || wy >= Q.oh) return;
  const uint8_t *__restrict__ src = frames.in[blockIdx.z] + Q.src_off;
  uint8_t *__restrict__ dst = frames.out[blockIdx.z] + Q.dst_off;
  unsigned o;
  if (Q.mode == PM_COPY) {
    o = __ldg ((const unsigned *) (src + (size_t) wy * Q.sstride) + wx);
    if (Q.swz) o = __byte_perm (o, 0, Q.swz);
  } else if (Q.mode == PM_HALVE_V) {
    o = avg_ceil4 (__ldg ((const unsigned *) (src + (size_t) (2 * wy) * Q.sstride) + wx),
        __ldg ((const unsigned *) (src + (size_t) (2 * wy + 1) * Q.sstride) + wx));
  } else if (Q.mode == PM_HALVE_H) {
    const uint2 a = __ldg ((const uint2 *) (src + (size_t) wy * Q.sstride) + wx);
    o = avg_ceil4 (__byte_perm (a.x, a.y, 0x6420), __byte_perm (a.x, a.y, 0x7531));
  } else {                                                         // PM_HALVE_HV: lines first, then the byte pairs
    const uint2 a = __ldg ((const uint2 *) (src + (size_t) (2 * wy) * Q.sstride) + wx);
    const uint2 b = __ldg ((const uint2 *) (src + (size_t) (2 * wy + 1) * Q.sstride) + wx);
    const unsigned t = avg_ceil4 (a.x, b.x), u = avg_ceil4 (a.y, b.y);
    o = avg_ceil4 (__byte_perm (t, u, 0x6420), __byte_perm (t, u, 0x7531));
  }
  *((unsigned *) (dst + (size_t) wy * Q.dstride) + wx) = o;
}

struct PlanesState {
  uint32_t *d_off[3][2] = {{nullptr}};
  int16_t *d_coef[3][2] = {{nullptr}};
  PlanesParams params;
  PlaneFastState fast[3];        // planes that run vcs_planes_fast_kernel instead (fast[i].ok)
  bool ready = false;
};

// slow: the byte-wise kernel for every plane (A/B knob B200_PLANES_SLOW)
inline int prepare_planes (const VcsPlan & p, PlanesState * st, bool slow)
{
  memset (&st->params, 0, sizeof (st->params));
  st->params.n_planes = p.n_planes;
  for (int i = 0; i < p.n_planes; i++) {
    const PlanePlan & q = p.planes[i];
    PlaneDev & d = st->params.pl[i];
    d.src_off = p.in.offset[q.src_plane]; d.dst_off = p.out.offset[i];
    d.sstride = p.in.stride[q.src_plane]; d.dstride = p.out.stride[i];
    d.iw = q.iw; d.ih = q.ih; d.ow = q.ow; d.oh = q.oh; d.ne = q.ne; d.mode = q.mode; d.h_first = q.h_first ? 1 : 0;
    d.swz = q.swz;
    {
      const bool hh = q.mode == PM_HALVE_H || q.mode == PM_HALVE_HV;     // these read 8 source bytes per 4 output bytes
      const int sa = hh ? 7 : 3;
      d.vec4 = ((q.ow * q.ne) & 3) == 0 && (d.dstride & 3) == 0 && (d.dst_off & 3) == 0 && (d.sstride & sa) == 0 &&
          (d.src_off & sa) == 0;
    }
    if (q.mode != PM_SCALE) continue;
    {
      std::vector<int32_t> hp, vp;
      const bool okf = !slow && plan_plane_fast (q, d.sstride, d.src_off, d.dstride, d.dst_off, &st->fast[i], &hp, &vp);
      if (okf) {
        const int s = prepare_plane_fast (q, hp, vp, &st->fast[i]);
        if (s != B200_OK) return s;
      }
    }
    const AxisPlan *ax[2] = {&q.h, &q.v};
    PlaneAxisDev *dv[2] = {&d.h, &d.v};
    for (int a = 0; a < 2; a++) {
      int s;
      if ((s = upload (&st->d_off[i][a], ax[a]->offset.data (), ax[a]->offset.size ())) != B200_OK) return s;
      if ((s = upload (&st->d_coef[i][a], ax[a]->coef.data (), ax[a]->coef.size ())) != B200_OK) return s;
      dv[a]->offset = st->d_off[i][a]; dv[a]->coef = st->d_coef[i][a];
      dv[a]->mode = ax[a]->mode; dv[a]->n_taps = ax[a]->n_taps;
    }
  }
  st->ready = true;
  return B200_OK;
}

inline void free_planes (PlanesState * st)
{
  for (int i = 0; i < 3; i++)
    for (int a = 0; a < 2; a++) { cudaFree (st->d_off[i][a]); cudaFree (st->d_coef[i][a]); }
  for (int i = 0; i < 3; i++) free_plane_fast (&st->fast[i]);
}

// plane i runs a launch of its own: a word-wide plan (vcs_planes_fast_kernel) or copy / halve of word-aligned rows
// (vcs_planes_vec_kernel); both need 8-byte aligned frames (`aligned`)
inline bool plane_own_launch (const PlanesState & st, int i, bool aligned)
{
  const PlaneDev & q = st.params.pl[i];
  return aligned && (st.fast[i].ok || (q.vec4 && q.mode != PM_SCALE && q.mode != PM_DOUBLE));
}

// the launches of launch_planes: one per plane with a launch of its own, one vcs_planes_kernel for the rest.  Unprepared
// (a host-only handle): one vcs_planes_kernel.
inline int plane_launches (const PlanesState & st, bool aligned)
{
  if (!st.ready) return 1;
  int own = 0;
  for (int i = 0; i < st.params.n_planes; i++) own += plane_own_launch (st, i, aligned) ? 1 : 0;
  return own + (own < st.params.n_planes ? 1 : 0);
}

// the kernel named for a plane-scaling handle: the first plane's word-wide kernel, else the byte-wise one
inline const char *planes_kernel_name (const PlanesState & st)
{
  for (int i = 0; i < st.params.n_planes; i++)
    if (st.fast[i].ok) return st.fast[i].vfirst ? "vcs_planes_fast_vfirst_kernel" : "vcs_planes_fast_kernel";
  return "vcs_planes_kernel";
}

inline int launch_planes (const PlanesState & st, const VcsBatch & batch, int n, cudaStream_t stream, bool aligned)
{
  PlanesParams P;
  memset (&P, 0, sizeof (P));
  for (int i = 0; i < st.params.n_planes; i++) {
    const PlaneDev & q = st.params.pl[i];
    if (!plane_own_launch (st, i, aligned)) {
      P.pl[P.n_planes++] = q;
    } else if (st.fast[i].ok) {
      const int s = launch_plane_fast (st.fast[i], batch, n, stream);
      if (s != B200_OK) return s;
    } else {
      const dim3 grid ((((q.ow * q.ne) >> 2) + 63) / 64, (q.oh + 3) / 4, n);
      vcs_planes_vec_kernel <<<grid, 256, 0, stream>>> (q, batch);
      B200_CUDA_TRY (cudaGetLastError ());
    }
  }
  if (P.n_planes == 0) return B200_OK;
  if (!aligned)
    for (int i = 0; i < P.n_planes; i++) P.pl[i].vec4 = 0;
  int wmax = 0, hmax = 0;
  for (int i = 0; i < P.n_planes; i++) {
    wmax = max (wmax, P.pl[i].ow * P.pl[i].ne);
    hmax = max (hmax, P.pl[i].oh);
  }
  const dim3 grid ((wmax + PL_TW - 1) / PL_TW, (hmax + PL_TH - 1) / PL_TH, P.n_planes * n);
  vcs_planes_kernel <<<grid, 256, 0, stream>>> (P, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

// packed RGB -> planar RGB (RGBP / BGRP).  The reference runs these pairs through its chain without a matrix stage: unpack
// to ARGB, the scalers, then pack_RGBP / pack_BGRP (gst-libs/gst/video/video-format.c:7496-7536), which store the R, G
// and B bytes of each ARGB pixel in their own planes and drop the alpha.  The scalers are the packed RGB ones above (4-byte
// pixels, into a per-handle scratch image); vcs_rgb_deinterleave_kernel is the pack.  YUV inputs never come here: their
// kernels store the three planes themselves (store_planar_px).
struct DeintDev {
  int w, h;
  unsigned long long soff;       // packed 4-byte pixels: the input frame (unchanged size) or the scaled scratch image
  int sstride;
  unsigned sel;                  // plane k takes source byte (sel >> 4k) & 3
  unsigned long long off[3];
  int stride[3];
};

struct DeintBatch {
  const uint8_t *src[B200_VCS_MAX_BATCH];
  uint8_t *out[B200_VCS_MAX_BATCH];
};

// one thread per pixel, 64 x 4 pixels per CTA: each warp reads 128 consecutive source bytes and writes 32 consecutive
// bytes of every plane
__global__ void __launch_bounds__ (256)
vcs_rgb_deinterleave_kernel (const DeintDev D, const DeintBatch frames)
{
  const int x = blockIdx.x * 64 + (threadIdx.x & 63), y = blockIdx.y * 4 + (threadIdx.x >> 6);
  if (x >= D.w || y >= D.h) return;
  const uint8_t *__restrict__ s = frames.src[blockIdx.z] + D.soff + (size_t) y * D.sstride + 4 * (size_t) x;
  uint8_t *__restrict__ o = frames.out[blockIdx.z];
#pragma unroll
  for (int k = 0; k < 3; k++) o[D.off[k] + (size_t) y * D.stride[k] + x] = s[(D.sel >> (4 * k)) & 3];
}

inline int launch_rgb_deinterleave (const DeintDev & d, const DeintBatch & b, int n, cudaStream_t stream)
{
  const dim3 grid ((d.w + 63) / 64, (d.h + 3) / 4, n);
  vcs_rgb_deinterleave_kernel <<<grid, 256, 0, stream>>> (d, b);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
