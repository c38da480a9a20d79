// gstreamer_b200/csrc/vcs_ntap.cuh — fused kernel for n-tap filters at ANY ratio (product code,
// sm_90a): 4:2:0 semi-planar -> packed RGB where at least one axis runs the reference's n-tap FIR
// (lanczos / cubic / sinc / linear-as-n-tap, video_scale_h_ntap_u8 + video_scale_v_ntap_u8) and the
// other one too or is untouched; horizontal pass first.  The exact-2:1 8-tap case has its own
// kernel (vcs_lanczos2.cuh); this one takes every other size, e.g. 1080p -> 720p or 4K -> 720p.
//
// Same arithmetic as vcs_generic_kernel stage by stage (see vcs_kernels.cuh for the citations):
//
//  A  shared with the light kernel (vcs_unpack_stage): byte-SIMD unpack + chroma up-sampling of
//     the tile's input region into three byte planes, 4 pixels per word
//  B  horizontal FIR: a thread owns one output column x 4 consecutive input lines x 3 channels.
//     Its taps are 8-bit and packed 4 per word (host table); the source bytes start at an arbitrary
//     column, so each tap word meets its 4 pixels through one funnel shift of two aligned words
//     (SHF.R.W) and one IDP.4A.U8.S8 — 3 instructions per 4 taps.  (acc+32)>>6 with saturation
//     packs the 4 lines of the column into ONE word (transposed), so that
//  C  the vertical FIR is the same loop over words of 4 lines: funnel shift by the window's line
//     offset, IDP.4A; then matrix (or not, when it ran first), alpha, byte order, coalesced store.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"
#include "vcs_device.h"
#include "vcs_kernels.cuh"
#include "vcs_lanczos2.cuh"      // packed-byte helpers
#include "vcs_light.cuh"         // stage A

namespace b200 {

struct NtapDev {
  int tw, th, rows, pitch;       // tile, staged rows (multiple of 4), words per staged row
  int ntw_h, ntw_v;              // packed tap words per output column / row
  const int *h_packed, *v_packed;
  int alpha_opaque;
  int std_pairs;                 // fast stage A (vcs_unpack_fast_cs) applies
};

constexpr int NTAP_THREADS = 256;

// NTW > 0: both n-tap axes use exactly NTW packed tap words (straight-line FIRs); NTW == 0: run-time loops
// PLOUT: planar RGB output (store_planar_px) instead of one 4-byte word per pixel
template <int HM, int VM, bool MFIRST, bool COSITED, int NTW, bool PLOUT = false>
__global__ void __launch_bounds__ (NTAP_THREADS, 2)
vcs_ntap_kernel (const VcsDev P, const NtapDev G, const VcsBatch frames)
{
  extern __shared__ __align__ (16) unsigned nsm[];
  const int ngr = G.rows / 4;                                    // staged groups of 4 input lines
  const int groups = ngr + 1 + G.ntw_v;                          // groups of the h-scaled tile (+ slack for padded taps)
  // S: [group][channel][word column][4 lines]  — the 4 lines of one word column are one uint4
  // T: [group][output column][channel (4)]     — one uint4 = the 3 channels' words (4 lines each)
  uint4 *S4 = (uint4 *) nsm;
  uint4 *T4 = S4 + ngr * 3 * G.pitch + 2;
  int *TH = (int *) (T4 + groups * G.tw);                        // [tw][ntw_h]
  int *TV = TH + G.tw * max (G.ntw_h, 1);                        // [th][ntw_v]
  unsigned *vrow = (unsigned *) (TV + G.th * max (G.ntw_v, 1));  // [th] first source line of each output row
  uint4 *ent = (uint4 *) (((uintptr_t) (vrow + G.th) + 15) & ~(uintptr_t) 15);   // [rows] entries + count
  const int tid = threadIdx.x;
  const uint8_t *__restrict__ in = frames.in[blockIdx.z];
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const uint8_t *__restrict__ plane_y = in + P.off_y;

  const int ox0 = blockIdx.x * G.tw, oy0 = blockIdx.y * G.th;
  const int tw = min (G.tw, P.ow - ox0), th = min (G.th, P.oh - oy0);
  const int cx0 = P.h.offset[ox0], cx1 = P.h.offset[ox0 + tw - 1] + P.h.span;
  const int ry0 = P.v.offset[oy0], ry1 = P.v.offset[oy0 + th - 1] + P.v.span;
  const int cxa = cx0 & ~3, R = ry1 - ry0, ng = (cx1 - cxa + 3) >> 2;

  // tap words and source lines of this tile's columns and rows
  if (HM == 3)
    for (int i = tid; i < tw * G.ntw_h; i += NTAP_THREADS) TH[i] = __ldg (G.h_packed + (size_t) ox0 * G.ntw_h + i);
  if (VM == 3)
    for (int i = tid; i < th * G.ntw_v; i += NTAP_THREADS) TV[i] = __ldg (G.v_packed + (size_t) oy0 * G.ntw_v + i);
  if (tid < th) vrow[tid] = P.v.offset[oy0 + tid] - (unsigned) ry0;

  // ---------------------------------------------------------------- A: unpack + chroma up-sample
  if (COSITED && !MFIRST && G.std_pairs) {                        // warp-uniform: a property of the plan
    vcs_unpack_fast_cs<false, 2> (P, in, cxa, cx1, ry0, R, (unsigned *) S4, G.pitch, 0);
  } else {
    vcs_unpack_worklist (P, ry0, R, ent, G.rows);
    __syncthreads ();
    vcs_unpack_stage<MFIRST, COSITED, 2> (P, plane_y, in, cxa, ng, ent, (int) ent[G.rows].x, (unsigned *) S4,
        G.pitch, 0);
  }
  __syncthreads ();

  // ---------------------------------------------------------------- B: horizontal pass
  const int tx = tid % G.tw, ph = tid / G.tw, nph = NTAP_THREADS / G.tw;   // tw is 32, 64 or 128
  if (tx < tw) {
    const int base = (int) P.h.offset[ox0 + tx] - cxa;
    const int wi = base >> 2, sh = (base & 3) * 8;
    const int RG = (R + 3) >> 2;
    const int *th_taps = TH + tx * G.ntw_h;
    for (int g = ph; g < RG; g += nph) {
      const uint4 *sp = S4 + g * 3 * G.pitch + wi;               // channel ch at sp + ch * pitch
      uint4 o;
      if (HM == 3) {
        int acc[3][4];
        uint4 lo[3];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
          lo[ch] = sp[ch * G.pitch];
#pragma unroll
          for (int i = 0; i < 4; i++) acc[ch][i] = 32;
        }
#define NTAP_H_STEP(W)                                                                          \
        do {                                                                                   \
          const int t = th_taps[W];                                                            \
          sp++;                                                                                \
          _Pragma ("unroll") for (int ch = 0; ch < 3; ch++) {                                  \
            const uint4 hi = sp[ch * G.pitch];                                                 \
            acc[ch][0] = dp4a_u8s8 (__funnelshift_r (lo[ch].x, hi.x, sh), t, acc[ch][0]);      \
            acc[ch][1] = dp4a_u8s8 (__funnelshift_r (lo[ch].y, hi.y, sh), t, acc[ch][1]);      \
            acc[ch][2] = dp4a_u8s8 (__funnelshift_r (lo[ch].z, hi.z, sh), t, acc[ch][2]);      \
            acc[ch][3] = dp4a_u8s8 (__funnelshift_r (lo[ch].w, hi.w, sh), t, acc[ch][3]);      \
            lo[ch] = hi;                                                                       \
          }                                                                                    \
        } while (0)
        if (NTW > 0) {
#pragma unroll
          for (int w = 0; w < NTW; w++) NTAP_H_STEP (w);
        } else {
#pragma unroll 1
          for (int w = 0; w < G.ntw_h; w++) NTAP_H_STEP (w);
        }
#undef NTAP_H_STEP
        // (acc+32)>>6 saturated to u8 (video-orc.orc:2474-2481); 4 lines of the column in one word
        o.x = pack_sat2 (acc[0][1] >> 6, acc[0][0] >> 6, pack_sat2 (acc[0][3] >> 6, acc[0][2] >> 6, 0u));
        o.y = pack_sat2 (acc[1][1] >> 6, acc[1][0] >> 6, pack_sat2 (acc[1][3] >> 6, acc[1][2] >> 6, 0u));
        o.z = pack_sat2 (acc[2][1] >> 6, acc[2][0] >> 6, pack_sat2 (acc[2][3] >> 6, acc[2][2] >> 6, 0u));
      } else {
        const unsigned s01 = (unsigned) (base & 3) | (unsigned) (4 + (base & 3)) << 4;
        const uint4 a = sp[0], b = sp[G.pitch], c = sp[2 * G.pitch];
        o.x = __byte_perm (__byte_perm (a.x, a.y, s01), __byte_perm (a.z, a.w, s01), 0x5410);
        o.y = __byte_perm (__byte_perm (b.x, b.y, s01), __byte_perm (b.z, b.w, s01), 0x5410);
        o.z = __byte_perm (__byte_perm (c.x, c.y, s01), __byte_perm (c.z, c.w, s01), 0x5410);
      }
      o.w = 0u;
      T4[g * G.tw + tx] = o;
    }
  }
  __syncthreads ();

  // ---------------------------------------------------------------- C: vertical pass, matrix, pack
  if (tx < tw) {
    const int ox = ox0 + tx;
    int ah = 255;
    if (!G.alpha_opaque) ah = alpha_pass (255, P.h, ox);
    uint8_t *dst = out + P.off_out + (size_t) (oy0 + ph) * P.stride_out + (size_t) ox * 4u;
    const size_t dstep = (size_t) P.stride_out * nph;
    for (int ty = ph; ty < th; ty += nph, dst += dstep) {
      const int rb = (int) vrow[ty];
      const uint4 *tp = T4 + (rb >> 2) * G.tw + tx;
      const int sh = (rb & 3) * 8;
      int c0, c1, c2;
      if (VM == 3) {
        c0 = c1 = c2 = 32;
        uint4 lo = *tp;
        const int *tv_taps = TV + ty * G.ntw_v;
#define NTAP_V_STEP(W)                                                                          \
        do {                                                                                   \
          const int t = tv_taps[W];                                                            \
          tp += G.tw;                                                                          \
          const uint4 hi = *tp;                                                                \
          c0 = dp4a_u8s8 (__funnelshift_r (lo.x, hi.x, sh), t, c0);                            \
          c1 = dp4a_u8s8 (__funnelshift_r (lo.y, hi.y, sh), t, c1);                            \
          c2 = dp4a_u8s8 (__funnelshift_r (lo.z, hi.z, sh), t, c2);                            \
          lo = hi;                                                                             \
        } while (0)
        if (NTW > 0) {
#pragma unroll
          for (int w = 0; w < NTW; w++) NTAP_V_STEP (w);
        } else {
#pragma unroll 1
          for (int w = 0; w < G.ntw_v; w++) NTAP_V_STEP (w);
        }
#undef NTAP_V_STEP
        c0 >>= 6; c1 >>= 6; c2 >>= 6;
      } else {
        const uint4 w = *tp;
        const unsigned sel = 0x4440u | (unsigned) (rb & 3);
        c0 = (int) __byte_perm (w.x, 0, sel); c1 = (int) __byte_perm (w.y, 0, sel); c2 = (int) __byte_perm (w.z, 0, sel);
      }
      int al = 255;
      if (!G.alpha_opaque) al = alpha_pass (ah, P.v, oy0 + ty);
      unsigned argb;
      if (MFIRST) {
        argb = pack_sat2 (c0, al, pack_sat2 (c2, c1, 0u));
      } else {
        argb = light_matrix (pack_sat2 (c1, c0, pack_sat2 (0, c2, 0u)), P);
        if (!G.alpha_opaque) argb = (argb & 0xffffff00u) | (unsigned) al;
      }
      if (PLOUT) store_planar_px (P, out, ox, oy0 + ty, __byte_perm (argb, 0, P.sel));
      else *(unsigned *) dst = __byte_perm (argb, 0, P.sel);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Vertical pass first (chain_scale picks it when out_w * in_h > in_w * out_h).
//  A   as above, into plain byte planes S[ch][line][word column]
//  B'  vertical FIR on two 16-bit lanes per register: acc += tap * (bytes 0,2) and tap * (bytes 1,3) with
//      32-bit IMAD — the low lane is exact modulo 2^16, the high lane is off by the low lane's borrow, which
//      bit 15 of the low lane gives back (|sums| < 2^15 is an eligibility condition).  One word = 4 columns.
//  C'  horizontal FIR per output pixel with funnel shift + IDP.4A on the v-scaled rows, matrix, pack.
template <int HM, int VM, bool MFIRST, bool COSITED, bool PLOUT = false>
__global__ void __launch_bounds__ (NTAP_THREADS, 2)
vcs_ntap_vfirst_kernel (const VcsDev P, const NtapDev G, const VcsBatch frames)
{
  extern __shared__ __align__ (16) unsigned nsm[];
  const int plane_words = G.rows * G.pitch, tplane = G.th * G.pitch;
  unsigned *S = nsm;                                             // [3][rows][pitch]
  unsigned *T = S + 3 * plane_words + 4;                         // [3][th][pitch]
  int *TH = (int *) (T + 3 * tplane + 4);                        // [tw][ntw_h]
  int *TV = TH + G.tw * max (G.ntw_h, 1);                        // [th][n_taps_v]  (16-bit taps, one per word)
  unsigned *vrow = (unsigned *) (TV + G.th * max (P.v.n_taps, 1));
  uint4 *ent = (uint4 *) (((uintptr_t) (vrow + G.th) + 15) & ~(uintptr_t) 15);
  const int tid = threadIdx.x, lane = tid & 31;
  const uint8_t *__restrict__ in = frames.in[blockIdx.z];
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const uint8_t *__restrict__ plane_y = in + P.off_y;

  const int ox0 = blockIdx.x * G.tw, oy0 = blockIdx.y * G.th;
  const int tw = min (G.tw, P.ow - ox0), th = min (G.th, P.oh - oy0);
  const int cx0 = P.h.offset[ox0], cx1 = P.h.offset[ox0 + tw - 1] + P.h.span;
  const int ry0 = P.v.offset[oy0], ry1 = P.v.offset[oy0 + th - 1] + P.v.span;
  const int cxa = cx0 & ~3, R = ry1 - ry0, ng = (cx1 - cxa + 3) >> 2;

  if (HM == 3)
    for (int i = tid; i < tw * G.ntw_h; i += NTAP_THREADS) TH[i] = __ldg (G.h_packed + (size_t) ox0 * G.ntw_h + i);
  if (VM == 3)
    for (int i = tid; i < th * P.v.n_taps; i += NTAP_THREADS) TV[i] = (int) P.v.coef[(size_t) oy0 * P.v.n_taps + i];
  if (tid < th) vrow[tid] = P.v.offset[oy0 + tid] - (unsigned) ry0;

  if (COSITED && !MFIRST && G.std_pairs) {
    vcs_unpack_fast_cs<false, 1> (P, in, cxa, cx1, ry0, R, S, G.pitch, plane_words);
  } else {
    vcs_unpack_worklist (P, ry0, R, ent, G.rows);
    __syncthreads ();
    vcs_unpack_stage<MFIRST, COSITED, 1> (P, plane_y, in, cxa, ng, ent, (int) ent[G.rows].x, S, G.pitch, plane_words);
  }
  __syncthreads ();

  // ---------------------------------------------------------------- B': vertical pass
  if (VM == 3) {
    const int nv = P.v.n_taps;
    for (int ty = tid >> 5; ty < th; ty += NTAP_THREADS / 32) {
      const int rb = (int) vrow[ty];
      const int *tv = TV + ty * nv;
      for (int j = lane; j < ng; j += 32) {
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
          const unsigned *sp = S + ch * plane_words + rb * G.pitch + j;
          unsigned ae = 0x00200020u, ao = 0x00200020u;           // +32 in every lane
#pragma unroll 2
          for (int k = 0; k < nv; k++) {
            const unsigned w = sp[k * G.pitch];
            const unsigned t = (unsigned) tv[k];
            ae += t * (w & 0x00ff00ffu);
            ao += t * __byte_perm (w, 0, 0x4341);
          }
          // lanes -> four signed sums (the high lane takes back the low lane's borrow), >> 6, saturate
          const int e0 = (int) (short) ae, e1 = ((int) ae >> 16) + (int) ((ae >> 15) & 1u);
          const int o0 = (int) (short) ao, o1 = ((int) ao >> 16) + (int) ((ao >> 15) & 1u);
          T[ch * tplane + ty * G.pitch + j] = pack_sat2 (o0 >> 6, e0 >> 6, pack_sat2 (o1 >> 6, e1 >> 6, 0u));
        }
      }
    }
    __syncthreads ();
  }

  // ---------------------------------------------------------------- C': horizontal pass, matrix, pack
  const int tx = tid % G.tw, ph = tid / G.tw, nph = NTAP_THREADS / G.tw;
  if (tx < tw) {
    const int ox = ox0 + tx;
    const int base = (int) P.h.offset[ox] - cxa;
    const int wi = base >> 2, sh = (base & 3) * 8;
    const int *th_taps = TH + tx * G.ntw_h;
    uint8_t *dst = out + P.off_out + (size_t) (oy0 + ph) * P.stride_out + (size_t) ox * 4u;
    const size_t dstep = (size_t) P.stride_out * nph;
    for (int ty = ph; ty < th; ty += nph, dst += dstep) {
      // the row this output line reads: v-scaled, or straight from the staged input when the vertical axis is a copy
      const unsigned *row = VM == 3 ? T + ty * G.pitch + wi : S + (int) vrow[ty] * G.pitch + wi;
      const int cstep = VM == 3 ? tplane : plane_words;
      int c[3];
      if (HM == 3) {
        unsigned lo[3];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) { c[ch] = 32; lo[ch] = row[ch * cstep]; }
#pragma unroll 1
        for (int w = 0; w < G.ntw_h; w++) {
          const int t = th_taps[w];
#pragma unroll
          for (int ch = 0; ch < 3; ch++) {
            const unsigned hi = row[ch * cstep + w + 1];
            c[ch] = dp4a_u8s8 (__funnelshift_r (lo[ch], hi, sh), t, c[ch]);
            lo[ch] = hi;
          }
        }
#pragma unroll
        for (int ch = 0; ch < 3; ch++) c[ch] >>= 6;
      } else {
        const unsigned sel = 0x4440u | (unsigned) (base & 3);
#pragma unroll
        for (int ch = 0; ch < 3; ch++) c[ch] = (int) __byte_perm (row[ch * cstep], 0, sel);
      }
      int al = 255;
      if (!G.alpha_opaque) {                                     // alpha follows the passes in their order: v, then h
        al = alpha_pass (255, P.v, oy0 + ty);
        al = alpha_pass (al, P.h, ox);
      }
      unsigned argb;
      if (MFIRST) {
        argb = pack_sat2 (c[0], al, pack_sat2 (c[2], c[1], 0u));
      } else {
        argb = light_matrix (pack_sat2 (c[1], c[0], pack_sat2 (0, c[2], 0u)), P);
        if (!G.alpha_opaque) argb = (argb & 0xffffff00u) | (unsigned) al;
      }
      if (PLOUT) store_planar_px (P, out, ox, oy0 + ty, __byte_perm (argb, 0, P.sel));
      else *(unsigned *) dst = __byte_perm (argb, 0, P.sel);
    }
  }
}

typedef void (*ntap_kernel_fn) (const VcsDev, const NtapDev, const VcsBatch);

template <int HM, int VM, int NTW, bool PLOUT>
inline ntap_kernel_fn ntap_kernel_pick_out (const VcsPlan & p)
{
  if (p.matrix_first) return p.h_cosited ? vcs_ntap_kernel<HM, VM, true, true, NTW, PLOUT> : vcs_ntap_kernel<HM, VM, true, false, NTW, PLOUT>;
  return p.h_cosited ? vcs_ntap_kernel<HM, VM, false, true, NTW, PLOUT> : vcs_ntap_kernel<HM, VM, false, false, NTW, PLOUT>;
}

template <int HM, int VM, int NTW>
inline ntap_kernel_fn ntap_kernel_pick (const VcsPlan & p)
{
  return p.rgbp_out ? ntap_kernel_pick_out<HM, VM, NTW, true> (p) : ntap_kernel_pick_out<HM, VM, NTW, false> (p);
}

template <int HM, int VM>
inline ntap_kernel_fn ntap_kernel_pick_ntw (const VcsPlan & p)
{
  switch (common_tap_words (HM, VM, p.ntw_h, p.ntw_v)) {
    case 1: return ntap_kernel_pick<HM, VM, 1> (p);
    case 2: return ntap_kernel_pick<HM, VM, 2> (p);
    case 3: return ntap_kernel_pick<HM, VM, 3> (p);
    case 4: return ntap_kernel_pick<HM, VM, 4> (p);
    default: return ntap_kernel_pick<HM, VM, 0> (p);
  }
}

template <int HM, int VM, bool PLOUT>
inline ntap_kernel_fn ntap_vfirst_pick_out (const VcsPlan & p)
{
  if (p.matrix_first) return p.h_cosited ? vcs_ntap_vfirst_kernel<HM, VM, true, true, PLOUT> : vcs_ntap_vfirst_kernel<HM, VM, true, false, PLOUT>;
  return p.h_cosited ? vcs_ntap_vfirst_kernel<HM, VM, false, true, PLOUT> : vcs_ntap_vfirst_kernel<HM, VM, false, false, PLOUT>;
}

template <int HM, int VM>
inline ntap_kernel_fn ntap_vfirst_pick (const VcsPlan & p)
{
  return p.rgbp_out ? ntap_vfirst_pick_out<HM, VM, true> (p) : ntap_vfirst_pick_out<HM, VM, false> (p);
}

inline ntap_kernel_fn ntap_kernel_for (const VcsPlan & p)
{
  if (!p.h_first) {
    if (p.h.mode == 3 && p.v.mode == 3) return ntap_vfirst_pick<3, 3> (p);
    if (p.h.mode == 3 && p.v.mode == 1) return ntap_vfirst_pick<3, 1> (p);
    if (p.h.mode == 1 && p.v.mode == 3) return ntap_vfirst_pick<1, 3> (p);
    return nullptr;
  }
  if (p.h.mode == 3 && p.v.mode == 3) return ntap_kernel_pick_ntw<3, 3> (p);
  if (p.h.mode == 3 && p.v.mode == 1) return ntap_kernel_pick_ntw<3, 1> (p);
  if (p.h.mode == 1 && p.v.mode == 3) return ntap_kernel_pick_ntw<1, 3> (p);
  return nullptr;
}

struct NtapState {
  int *d_h = nullptr, *d_v = nullptr;
  bool ready = false;
};

inline int prepare_ntap (const VcsPlan & p, NtapState * st)
{
  int s;
  if ((s = upload (&st->d_h, p.h_packed.data (), p.h_packed.size ())) != B200_OK) return s;
  if ((s = upload (&st->d_v, p.v_packed.data (), p.v_packed.size ())) != B200_OK) return s;
  if ((s = allow_max_dyn_smem (ntap_kernel_for (p))) != B200_OK) return s;
  st->ready = true;
  return B200_OK;
}

inline int launch_ntap (const VcsDev & dev, const VcsPlan & p, const NtapState & st, const VcsBatch & batch, int n,
    cudaStream_t stream)
{
  ntap_kernel_fn fn = ntap_kernel_for (p);
  if (!fn) return B200_ERR_STATE;
  NtapDev g;
  g.tw = p.ntap_tw; g.th = p.ntap_th; g.rows = p.ntap_rows; g.pitch = p.ntap_pitch;
  g.ntw_h = p.ntw_h; g.ntw_v = p.ntw_v; g.h_packed = st.d_h; g.v_packed = st.d_v;
  g.alpha_opaque = p.ntap_alpha_opaque ? 1 : 0;
  g.std_pairs = p.light_std_pairs ? 1 : 0;
  for (int i = 0; i < n; i++) if (((uintptr_t) batch.in[i]) & 7) g.std_pairs = 0;     // the fast stage A loads 64 bits at a time
  dim3 grid ((p.out.width + g.tw - 1) / g.tw, (p.out.height + g.th - 1) / g.th, n);
  fn <<<grid, NTAP_THREADS, p.ntap_smem, stream>>> (dev, g, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
