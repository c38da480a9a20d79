// gstreamer_b200/csrc/vcs_lanczos2_v2.cuh — second form of the headline kernel (product code, sm_90a).
//
// Same tile, same two phases and the same arithmetic as vcs_lanczos2_kernel<true, 4, 60, 1, true> (vcs_lanczos2.cuh, which
// stays the fallback for every plan this one does not take); what changes is what the SASS histogram of that kernel showed
// to be overhead (the kernel is bound by the issue slots and the integer pipe):
//
//  * interior tiles (no frame border in reach: most tiles of a 4K frame) have ONE set of taps for every column - the
//    plan proves it on the host - so the taps are kernel constants (constant-bank operands of IDP.4A): no table loads, twelve
//    registers less
//  * chroma words are built shifted by one pixel ([o0 e1 o1 e2] instead of [e0 o0 e1 o1]; the same PRMTs with the shifted
//    sample word as the second source), which puts the four output columns' windows on the 0/2/4/6 byte grid: 10 IDP.4A per
//    line and channel instead of 12 (two tap words are all zero and never issued).  Luma comes from memory on the 8-byte
//    grid and keeps 12.
//  * a warp's line groups are consecutive: the chroma row two groups share is up-sampled once and carried in registers, and
//    the next group's six loads are issued before the current group's arithmetic (the H phase spent 2.3 stalled warps per
//    issue waiting for its loads)
//  * V phase: accumulators preset to 128 - 32768 and packed with signed 16-bit saturation, so byte 1 of each half IS the
//    rounded, saturated sample minus 128 - the bias xor and the byte-gather PRMT go, the third channel of two pixels shares
//    one pack; uniform row groups take their taps from constants and skip their two all-zero tap words; the output byte
//    order is the ARGUMENT order of the two saturating packs (template SEL) instead of a final PRMT.
//
// Reference semantics as in vcs_lanczos2.cuh / vcs_kernels.cuh (video-converter.c chain, video-scaler.c:621-760, :986-1072,
// video-orc.orc:2388-2481, :1634-1688).
#pragma once

#include "vcs_lanczos2.cuh"

namespace b200 {

struct Lanczos2V2Dev {
  int hy[6], hc[6], vv[6];             // uniform taps times 4: first half of an L2_FIR4 table row (luma frame, chroma frame, vertical)
  const uint8_t *vkind;                // per row group: 2 uniform (vv), 1 table times 4, 0 plain table
};

__device__ __forceinline__ unsigned pack_sat_s16x2 (int a, int b)     // { sat_s16 (a), sat_s16 (b) }, b in the low half
{
#ifdef B200_CUDA_EMU
  return ((unsigned) (min (max (a, -32768), 32767) & 0xffff) << 16) | (unsigned) (min (max (b, -32768), 32767) & 0xffff);
#else
  unsigned d;
  asm ("cvt.pack.sat.s16.s32 %0, %1, %2;" : "=r" (d) : "r" (a), "r" (b));
  return d;
#endif
}

// constants K[6]: the first half of an L2_FIR4 table row - with one set of taps for every output the second half (outputs 2, 3
// on words 1..3) repeats the first (outputs 0, 1 on words 0..2), which the host verifies; Z: word 2 is zero (windows on the
// 0/2/4/6 byte grid)
#define L2_FIR4K(o0, o1, o2, o3, w0, w1, w2, w3, K, INIT, Z)                                    \
  do {                                                                                         \
    o0 = dp4a_u8s8 (w1, K[1], dp4a_u8s8 (w0, K[0], INIT));                                     \
    if (!(Z)) o0 = dp4a_u8s8 (w2, K[2], o0);                                                   \
    o1 = dp4a_u8s8 (w2, K[5], dp4a_u8s8 (w1, K[4], dp4a_u8s8 (w0, K[3], INIT)));               \
    o2 = dp4a_u8s8 (w2, K[1], dp4a_u8s8 (w1, K[0], INIT));                                     \
    if (!(Z)) o2 = dp4a_u8s8 (w3, K[2], o2);                                                   \
    o3 = dp4a_u8s8 (w3, K[5], dp4a_u8s8 (w2, K[4], dp4a_u8s8 (w1, K[3], INIT)));               \
  } while (0)
#define L2_FIR4T(o0, o1, o2, o3, w0, w1, w2, w3, T, INIT)                                      \
  do {                                                                                         \
    o0 = dp4a_u8s8 (w2, T[0].z, dp4a_u8s8 (w1, T[0].y, dp4a_u8s8 (w0, T[0].x, INIT)));         \
    o1 = dp4a_u8s8 (w2, T[1].y, dp4a_u8s8 (w1, T[1].x, dp4a_u8s8 (w0, T[0].w, INIT)));         \
    o2 = dp4a_u8s8 (w3, T[2].x, dp4a_u8s8 (w2, T[1].w, dp4a_u8s8 (w1, T[1].z, INIT)));         \
    o3 = dp4a_u8s8 (w3, T[2].w, dp4a_u8s8 (w2, T[2].z, dp4a_u8s8 (w1, T[2].y, INIT)));         \
  } while (0)

// SEL: the output format's byte selector (VcsDev::sel) when known at compile time, -1: applied with a PRMT per pixel.
// PF: 0, nothing else exists any more (the H phase always loads one line group ahead); MINB, PF, TH and NT stay in the
// argument list because the instantiation's full name is what the recorded route table (tests/golden/vcs_routes.json) holds.
// PLANAR: I420 / YV12 input - a chroma row is one 32-bit word from each of the U and V planes (already de-interleaved).
// YUVOUT: 4:2:0 output through the chain (VcsDev::yuv_out): no matrix stage, {255, Y, U, V} pixels for vcs_down420_kernel.
// PLOUT: planar RGB output (RGBP / BGRP): the packed pixel's bytes 0..2 go to three planes (store_planar_px).
// TH x NT: output rows per tile and threads per CTA: 60 x 256 at MINB = 4 CTAs per SM (124 x 512 at 2 measured slower on H100).
template <int MINB, int SEL, int PF, int TH = 60, int NT = L2_THREADS, bool PLANAR = false, bool YUVOUT = false, bool PLOUT = false>
__global__ void __launch_bounds__ (NT, MINB)
vcs_lanczos2_v2_kernel (const VcsDev P, const Lanczos2Dev L, const Lanczos2V2Dev K, const VcsBatch frames)
{
  static_assert (PF == 0, "one H-phase load schedule");
  constexpr int NWC = 1, NWARP = NT / 32;
  constexpr int L2_NG = L2Shape<TH, NWC>::NG, L2_TW = L2Shape<TH, NWC>::TW, L2_TWP = L2Shape<TH, NWC>::TWP;

  extern __shared__ __align__ (16) unsigned hs[];                // [3][L2_NG][L2_TWP] words
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync (0xffffffffu, (int) (threadIdx.x >> 5), 0);
  const uint8_t *__restrict__ in = frames.in[blockIdx.z];
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const uint8_t *__restrict__ plane_y = in + P.off_y;
  const uint8_t *__restrict__ plane_c = in + P.off_c;
  const uint8_t *__restrict__ plane_u = in + P.off_u, *__restrict__ plane_v = in + P.off_v;   // PLANAR
  const int x0 = blockIdx.x * L2_TW, oy0 = blockIdx.y * TH;
  const int R0 = 2 * oy0 - 3;                                    // first input line of the tile
  const int crows = P.ih >> 1;
  const unsigned selU = P.u_index ? 0x7531u : 0x6420u, selV = P.u_index ? 0x6420u : 0x7531u;

  // ---------------------------------------------------------------- H phase
  // line groups this tile's rows need (the frame's last tile row may be short)
  const int ng = min (L2_NG, (2 * min (TH, P.oh - oy0) + 6 + 3) >> 2);
  // tiles at the left / right frame border take the table path (folded taps, clamped columns); tiles that only reach the top or
  // bottom border keep the constant taps and clamp their line / chroma-row indices
  const bool edge_tile = x0 == 0 || x0 + L2_TW + 4 >= P.ow;
  const bool edge_rows = R0 < 0 || R0 + 4 * ng > P.ih;

#define L2_PACK4X(A, c) __byte_perm (pack_sat_u16x2 (A[1][c], A[0][c]), pack_sat_u16x2 (A[3][c], A[2][c]), 0x7531)
#define L2_PACK4P(A, c) pack_sat2 (sra6 (A[1][c]), sra6 (A[0][c]), pack_sat2 (sra6 (A[3][c]), sra6 (A[2][c]), 0u))
#define L2_STOREV(ch, A, PACK)                                                                 \
    do {                                                                                       \
      uint4 o;                                                                                 \
      o.x = PACK (A, 0); o.y = PACK (A, 1); o.z = PACK (A, 2); o.w = PACK (A, 3);              \
      *(uint4 *) (hs + ((ch) * L2_NG + g) * L2_TWP + lane * 4) = o;                            \
    } while (0)
  // (3x+y+2)>>2 == avg_ceil (x, avg_floor (x,y)) on rows (a,b) -> lines 0,1 and (b,c) -> lines 2,3 (video-orc.orc:2705-2735)
#define L2_VPAIRS(D, lo, hi)                                                                   \
    do {                                                                                       \
      unsigned f;                                                                              \
      f = avg_floor4 (lo[0], lo[1]); D[0][0] = avg_ceil4 (lo[0], f); D[1][0] = avg_ceil4 (lo[1], f); \
      f = avg_floor4 (hi[0], hi[1]); D[0][1] = avg_ceil4 (hi[0], f); D[1][1] = avg_ceil4 (hi[1], f); \
      f = avg_floor4 (lo[1], lo[2]); D[2][0] = avg_ceil4 (lo[1], f); D[3][0] = avg_ceil4 (lo[2], f); \
      f = avg_floor4 (hi[1], hi[2]); D[2][1] = avg_ceil4 (hi[1], f); D[3][1] = avg_ceil4 (hi[2], f); \
    } while (0)

  if (edge_tile) {
    // tiles at a frame border: clamped lines / chroma rows / columns, per-column tap tables (folded taps do not fit times 4)
    const int4 *__restrict__ htab = L.htab;
    for (int item = warp; item < ng; item += NWARP) {
      const int g = item;
      const int col0 = x0 + (lane - 1) * 4;
      int4 T[3];
      {
        const int grp = min (max (col0 >> 2, 0), (P.ow >> 2) - 1);
        T[0] = __ldg (htab + grp * 3 + 0); T[1] = __ldg (htab + grp * 3 + 1); T[2] = __ldg (htab + grp * 3 + 2);
      }
      const int xb = min (max (2 * col0, 0), P.iw - 8);
      const bool right_edge = 2 * col0 + 8 >= P.iw;              // no chroma sample to the right
      const int y0 = R0 + 4 * g, m2 = (y0 - 1) >> 1;
      unsigned ulo[3], uhi[3], vlo[3], vhi[3];
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const int cr = min (max (m2 + k, 0), crows - 1);
        unsigned ue, ve;
        if (PLANAR) {
          ue = __ldg ((const unsigned *) (plane_u + (size_t) cr * P.stride_u + (xb >> 1)));
          ve = __ldg ((const unsigned *) (plane_v + (size_t) cr * P.stride_v + (xb >> 1)));
        } else {
          const uint2 c = __ldg ((const uint2 *) (plane_c + (size_t) cr * P.stride_c + xb));
          ue = __byte_perm (c.x, c.y, selU); ve = __byte_perm (c.x, c.y, selV);
        }
        unsigned un = __shfl_down_sync (0xffffffffu, ue, 1), vn = __shfl_down_sync (0xffffffffu, ve, 1);
        un = right_edge ? __byte_perm (ue, ue, 0x3321) : __byte_perm (ue, un, 0x4321);
        vn = right_edge ? __byte_perm (ve, ve, 0x3321) : __byte_perm (ve, vn, 0x4321);
        const unsigned uo = avg_ceil4 (ue, un), vo = avg_ceil4 (ve, vn);
        ulo[k] = __byte_perm (ue, uo, 0x5140); uhi[k] = __byte_perm (ue, uo, 0x7362);
        vlo[k] = __byte_perm (ve, vo, 0x5140); vhi[k] = __byte_perm (ve, vo, 0x7362);
      }
      unsigned U[4][2], V[4][2];
      L2_VPAIRS (U, ulo, uhi);
      L2_VPAIRS (V, vlo, vhi);
      int acc[4][4];
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const unsigned w0 = __shfl_up_sync (0xffffffffu, U[r][1], 1), w3 = __shfl_down_sync (0xffffffffu, U[r][0], 1);
        L2_FIR4T (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, U[r][0], U[r][1], w3, T, 32);
      }
      L2_STOREV (1, acc, L2_PACK4P);
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const unsigned w0 = __shfl_up_sync (0xffffffffu, V[r][1], 1), w3 = __shfl_down_sync (0xffffffffu, V[r][0], 1);
        L2_FIR4T (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, V[r][0], V[r][1], w3, T, 32);
      }
      L2_STOREV (2, acc, L2_PACK4P);
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int y = min (max (y0 + r, 0), P.ih - 1);
        const uint2 yy = __ldg ((const uint2 *) (plane_y + (size_t) y * P.stride_y + xb));
        const unsigned w0 = __shfl_up_sync (0xffffffffu, yy.y, 1), w3 = __shfl_down_sync (0xffffffffu, yy.x, 1);
        L2_FIR4T (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, yy.x, yy.y, w3, T, 32);
      }
      L2_STOREV (0, acc, L2_PACK4P);
    }
  } else {
    // interior tiles: uniform taps times 4 from the constant bank, chroma on the shifted grid, loads one item ahead
    const int xb = 2 * (x0 + (lane - 1) * 4);                    // byte column of the lane's 8 input pixels
    struct Raw { uint2 c[2]; uint2 y[4]; };
    // one chroma row: 8 interleaved bytes, or (PLANAR) .x = 4 U samples, .y = 4 V samples
    auto h_load_c = [&] (auto clamp_tag, int row) {
      const int cr = decltype (clamp_tag)::value ? min (max (row, 0), crows - 1) : row;
      if (PLANAR) {
        uint2 c;
        c.x = __ldg ((const unsigned *) (plane_u + (ptrdiff_t) cr * P.stride_u + (xb >> 1)));
        c.y = __ldg ((const unsigned *) (plane_v + (ptrdiff_t) cr * P.stride_v + (xb >> 1)));
        return c;
      }
      return __ldg ((const uint2 *) (plane_c + (ptrdiff_t) cr * P.stride_c + xb));
    };
    // what line group g needs beyond the chroma row it shares with group g - 1: two chroma rows and four lines
    auto h_load = [&] (auto clamp_tag, int g, Raw & r) {
      const int y0 = R0 + 4 * g, m2 = (y0 - 1) >> 1;
      r.c[0] = h_load_c (clamp_tag, m2 + 1); r.c[1] = h_load_c (clamp_tag, m2 + 2);
      if (decltype (clamp_tag)::value) {
#pragma unroll
        for (int k = 0; k < 4; k++)
          r.y[k] = __ldg ((const uint2 *) (plane_y + (size_t) min (max (y0 + k, 0), P.ih - 1) * P.stride_y + xb));
      } else {
        const uint8_t *py = plane_y + (ptrdiff_t) y0 * P.stride_y + xb;
#pragma unroll
        for (int k = 0; k < 4; k++) { r.y[k] = __ldg ((const uint2 *) py); py += P.stride_y; }
      }
    };
    // a chroma row up-sampled horizontally: [o0 e1 o1 e2], [o2 e3 o3 e4] of each plane, pixels 8L+1 .. 8L+8
    auto h_up = [&] (const uint2 c, unsigned & ulo, unsigned & uhi, unsigned & vlo, unsigned & vhi) {
      const unsigned ue = PLANAR ? c.x : __byte_perm (c.x, c.y, selU), ve = PLANAR ? c.y : __byte_perm (c.x, c.y, selV);
      unsigned un = __shfl_down_sync (0xffffffffu, ue, 1), vn = __shfl_down_sync (0xffffffffu, ve, 1);
      un = __byte_perm (ue, un, 0x4321);
      vn = __byte_perm (ve, vn, 0x4321);
      const unsigned uo = avg_ceil4 (ue, un), vo = avg_ceil4 (ve, vn);
      ulo = __byte_perm (uo, un, 0x5140); uhi = __byte_perm (uo, un, 0x7362);
      vlo = __byte_perm (vo, vn, 0x5140); vhi = __byte_perm (vo, vn, 0x7362);
    };
    auto h_item = [&] (int g, const unsigned (&ulo)[3], const unsigned (&uhi)[3], const unsigned (&vlo)[3], const unsigned (&vhi)[3],
        const uint2 (&ry)[4]) {
      unsigned U[4][2], V[4][2];
      L2_VPAIRS (U, ulo, uhi);
      L2_VPAIRS (V, vlo, vhi);
      int acc[4][4];
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const unsigned w0 = __shfl_up_sync (0xffffffffu, U[r][1], 1), w3 = __shfl_down_sync (0xffffffffu, U[r][0], 1);
        L2_FIR4K (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, U[r][0], U[r][1], w3, K.hc, 128, true);
      }
      L2_STOREV (1, acc, L2_PACK4X);
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const unsigned w0 = __shfl_up_sync (0xffffffffu, V[r][1], 1), w3 = __shfl_down_sync (0xffffffffu, V[r][0], 1);
        L2_FIR4K (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, V[r][0], V[r][1], w3, K.hc, 128, true);
      }
      L2_STOREV (2, acc, L2_PACK4X);
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const unsigned w0 = __shfl_up_sync (0xffffffffu, ry[r].y, 1), w3 = __shfl_down_sync (0xffffffffu, ry[r].x, 1);
        L2_FIR4K (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, ry[r].x, ry[r].y, w3, K.hy, 128, false);
      }
      L2_STOREV (0, acc, L2_PACK4X);
    };
    // a warp takes a run of consecutive line groups: the last chroma row of a group (rows m2, m2 + 1, m2 + 2) is the first of
    // the next (m2 + 2 ..), so its up-sampled words stay in registers and every group after the run's first loads and
    // up-samples two rows instead of three (a clamped row index that repeats is still the same row)
    auto h_run = [&] (auto clamp_tag) {
      const int per = (ng + NWARP - 1) / NWARP;                  // ng < L2_NG in the frame's last, short tile row
      const int g0 = warp * per, g1 = min (ng, g0 + per);
      if (g0 >= g1) return;
      // every load is issued before the arithmetic that precedes its use: the run's first chroma row and first group before
      // anything else, then each next group's six loads before the current group's FIRs
      const uint2 c0 = h_load_c (clamp_tag, (R0 + 4 * g0 - 1) >> 1);
      Raw r;
      h_load (clamp_tag, g0, r);
      unsigned ulo[3], uhi[3], vlo[3], vhi[3];
      h_up (c0, ulo[2], uhi[2], vlo[2], vhi[2]);
      for (int g = g0; g < g1; g++) {
        ulo[0] = ulo[2]; uhi[0] = uhi[2]; vlo[0] = vlo[2]; vhi[0] = vhi[2];
        h_up (r.c[0], ulo[1], uhi[1], vlo[1], vhi[1]);
        h_up (r.c[1], ulo[2], uhi[2], vlo[2], vhi[2]);
        Raw n;
        if (g + 1 < g1) h_load (clamp_tag, g + 1, n);
        h_item (g, ulo, uhi, vlo, vhi, r.y);
        r = n;
      }
    };
    if (edge_rows) h_run (std::true_type {}); else h_run (std::false_type {});
  }
  __syncthreads ();

  // ---------------------------------------------------------------- V phase
  // a warp owns output rows oy0+4q .. +3 for all columns of the tile; the row group's kind is warp-uniform and taken as a
  // branch between instantiations
  auto v_rows = [&] (auto kind_tag, int q) {
    constexpr int KIND = decltype (kind_tag)::value;             // 2 uniform constants, 1 table times 4, 0 plain table
    const int oy = oy0 + 4 * q;
    int4 T[3];
    if (KIND != 2) {
      const int4 *__restrict__ vtab = KIND == 1 ? L.vtab4 : L.vtab;
      T[0] = __ldg (vtab + (oy >> 2) * 3 + 0);
      T[1] = __ldg (vtab + (oy >> 2) * 3 + 1);
      T[2] = __ldg (vtab + (oy >> 2) * 3 + 2);
    }
    constexpr int vinit = KIND ? 128 - 32768 : 32;
    uint8_t *rowp[4];                                            // oh % 4 == 0: all 4 rows exist
    rowp[0] = out + P.off_out + (size_t) oy * P.stride_out + (size_t) (x0 + lane) * 4u;
#pragma unroll
    for (int i = 1; i < 4; i++) rowp[i] = rowp[i - 1] + P.stride_out;
#pragma unroll
    for (int k = 0; k < (L2_TW + 31) / 32; k++) {
      const int c = lane + 32 * k;
      const int ox = x0 + c;
      if ((32 * k + 32 <= L2_TW || c < L2_TW) && ox < P.ow) {
        const int sc = c + 4;                                    // smem column of this output column
        int a[3][4];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
          const unsigned *p = hs + (ch * L2_NG + 2 * q) * L2_TWP + sc;
          const unsigned w0 = p[0], w1 = p[L2_TWP], w2 = p[2 * L2_TWP], w3 = p[3 * L2_TWP];
          if (KIND == 2) L2_FIR4K (a[ch][0], a[ch][1], a[ch][2], a[ch][3], w0, w1, w2, w3, K.vv, vinit, true);
          else L2_FIR4T (a[ch][0], a[ch][1], a[ch][2], a[ch][3], w0, w1, w2, w3, T, vinit);
        }
        unsigned pv[2];
        if (KIND) { pv[0] = pack_sat_s16x2 (a[2][1], a[2][0]); pv[1] = pack_sat_s16x2 (a[2][3], a[2][2]); }
#pragma unroll
        for (int i = 0; i < 4; i++) {
          if (YUVOUT) {                                            // the scaled samples themselves: undo the -128 bias of the packs
            unsigned px;
            if (KIND) {
              const unsigned pyu = pack_sat_s16x2 (a[1][i], a[0][i]);
              px = (__byte_perm (pyu, pv[i >> 1], (i & 1) ? 0x7310u : 0x5310u) ^ 0x80808000u) | 0xffu;
            } else {
              px = __byte_perm (pack_sat2 (a[1][i] >> 6, a[0][i] >> 6, pack_sat2 (0, a[2][i] >> 6, 0u)), 0x000000ffu, 0x2104);
            }
            *(unsigned *) (rowp[i] + 128 * k) = px;
            continue;
          }
          int wy, wu, wv;
          if (KIND) {
            // byte 1 of sat_s16 (4 acc + 128 - 32768) = clamp ((acc + 32) >> 6, 0, 255) - 128: the biased sample, sign-splat to s16
            const unsigned pyu = pack_sat_s16x2 (a[1][i], a[0][i]);
            wy = prmt_s (pyu, 0x9911u); wu = prmt_s (pyu, 0xbb33u);
            wv = prmt_s (pv[i >> 1], (i & 1) ? 0xbb33u : 0x9911u);
          } else {
            unsigned yuv = pack_sat2 (a[1][i] >> 6, a[0][i] >> 6, pack_sat2 (0, a[2][i] >> 6, 0u));
            yuv ^= 0x00808080u;
            wy = prmt_s (yuv, 0x8800u); wu = prmt_s (yuv, 0x9911u); wv = prmt_s (yuv, 0xaa22u);
          }
          const int ty = ((wy * P.p1) >> 16) + 128;
          const int r = ty + ((wv * P.p2) >> 16);
          const int b = ty + ((wu * P.p3) >> 16);
          const int gg = ty + ((wu * P.p4) >> 16) + ((wv * P.p5) >> 16);
          unsigned px;
          if (SEL >= 0) {
            // output byte i <- component (SEL >> 4i) & 3 of (A, R, G, B): the order of the pack arguments
            const int comp[4] = {255, r, gg, b};
            px = pack_sat2 (comp[(SEL >> 4) & 3], comp[SEL & 3], pack_sat2 (comp[(SEL >> 12) & 3], comp[(SEL >> 8) & 3], 0u));
          } else {
            px = __byte_perm (pack_sat2 (r, 255, pack_sat2 (b, gg, 0u)), 0, P.sel);
          }
          if (PLOUT) store_planar_px (P, out, ox, oy + i, px);
          else *(unsigned *) (rowp[i] + 128 * k) = px;
        }
      }
    }
  };
  // Two more things were built, measured or checked, and dropped: (1) packing the 24 left-over
  // columns of the tile's 15 row groups into 12 full warp passes instead of 15 three-quarter-full ones - the packed passes'
  // per-lane row pointers and indices cost more than the three passes saved; (2) running the
  // left / right border tiles on the constant taps over edge-REPLICATED samples - the reference folds its edge taps in
  // double precision BEFORE quantising them, so the folded integer taps are not the uniform integer taps summed over the
  // replicated positions (column 1 of the bench shape: -3 8 28 28 7 -3 -1 against -4 8 28 28 8 -3 -1): not bit-exact.
  for (int q = warp; q < TH / 4; q += NWARP) {
    const int oy = oy0 + 4 * q;
    if (oy < P.oh) {
      const int kind = __ldg (K.vkind + (oy >> 2));
      if (kind == 2) v_rows (std::integral_constant<int, 2> {}, q);
      else if (kind == 1) v_rows (std::integral_constant<int, 1> {}, q);
      else v_rows (std::integral_constant<int, 0> {}, q);
    }
  }
#undef L2_PACK4X
#undef L2_PACK4P
#undef L2_STOREV
#undef L2_VPAIRS
}

// ------------------------------------------------------------------------------------ host side
struct Lanczos2V2Tables {
  bool ok = false;
  int hy[6], hc[6], vv[6];
  std::vector<uint8_t> vkind;
};

// the v2 kernel's preconditions on top of build_lanczos2_tables: taps times 4 everywhere the interior code looks, and one
// set of taps for all of those columns / the flagged row groups
inline Lanczos2V2Tables build_lanczos2_v2_tables (const VcsPlan & p, const Lanczos2Tables & t)
{
  Lanczos2V2Tables r;
  if (!t.ok || !t.x4_ok || !t.alpha_opaque) return r;
  std::vector<int> hc4; std::vector<uint8_t> hcfits;
  if (!pack_axis_lanczos2 (p.h, 3, &hc4, 4, &hcfits)) return r;  // the chroma frame: windows on the 0/2/4/6 byte grid
  const int groups = p.out.width / 4, ow = p.out.width, TW = L2_WCOLS;
  const int gm = groups / 2;
  if (!t.h4[gm] || !hcfits[gm] || hc4[(size_t) gm * 12 + 2] != 0) return r;
  for (int w = 0; w < 6; w++)                                    // outputs 2, 3 = outputs 0, 1 one word further
    if (t.htab4[(size_t) gm * 12 + w] != t.htab4[(size_t) gm * 12 + 6 + w] || hc4[(size_t) gm * 12 + w] != hc4[(size_t) gm * 12 + 6 + w]) return r;
  for (int x0 = TW; x0 + TW + 4 < ow; x0 += TW)                  // interior tile columns (the kernel's edge_tile test)
    for (int g = x0 / 4 - 1; g <= (x0 + TW) / 4; g++) {
      if (g < 0 || g >= groups || !t.h4[g] || !hcfits[g]) return r;
      for (int w = 0; w < 12; w++)
        if (t.htab4[(size_t) g * 12 + w] != t.htab4[(size_t) gm * 12 + w] || hc4[(size_t) g * 12 + w] != hc4[(size_t) gm * 12 + w]) return r;
    }
  const int vgroups = p.out.height / 4, vm = vgroups / 2;
  bool vuni = t.v4[vm] && t.vtab4[(size_t) vm * 12 + 2] == 0;
  for (int w = 0; w < 6; w++) vuni = vuni && t.vtab4[(size_t) vm * 12 + w] == t.vtab4[(size_t) vm * 12 + 6 + w];
  r.vkind.assign (vgroups, 0);
  for (int g = 0; g < vgroups; g++) {
    if (!t.v4[g]) continue;
    r.vkind[g] = 1;
    bool same = vuni;
    for (int w = 0; w < 12 && same; w++) same = t.vtab4[(size_t) g * 12 + w] == t.vtab4[(size_t) vm * 12 + w];
    if (same) r.vkind[g] = 2;
  }
  for (int w = 0; w < 6; w++) {
    r.hy[w] = t.htab4[(size_t) gm * 12 + w]; r.hc[w] = hc4[(size_t) gm * 12 + w]; r.vv[w] = t.vtab4[(size_t) vm * 12 + w];
  }
  r.ok = true;
  return r;
}

struct Lanczos2V2State {
  Lanczos2V2Dev dev;
  uint8_t *d_vkind = nullptr;
  bool ready = false;
};

inline int prepare_lanczos2_v2 (const Lanczos2V2Tables & t, Lanczos2V2State * st)
{
  int rc;
  if ((rc = upload (&st->d_vkind, t.vkind.data (), t.vkind.size ())) != B200_OK) return rc;
  for (int w = 0; w < 6; w++) { st->dev.hy[w] = t.hy[w]; st->dev.hc[w] = t.hc[w]; st->dev.vv[w] = t.vv[w]; }
  st->dev.vkind = st->d_vkind;
  st->ready = true;
  return B200_OK;
}

template <int SEL, bool PLANAR = false, bool YUVOUT = false, bool PLOUT = false>
inline int launch_lanczos2_v2_sel (const VcsDev & d, const Lanczos2State & st, const Lanczos2V2State & v2, const VcsBatch & batch,
    int n, cudaStream_t stream)
{
  constexpr int TH = 60, NT = L2_THREADS;
  auto kern = vcs_lanczos2_v2_kernel<4, SEL, 0, TH, NT, PLANAR, YUVOUT, PLOUT>;
  static bool attr_done[16] = {false};
  int dev = 0; cudaGetDevice (&dev);
  if (!attr_done[dev & 15]) {
    B200_CUDA_TRY (cudaFuncSetAttribute (kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L2Shape<TH, 1>::SMEM));
    attr_done[dev & 15] = true;
  }
  dim3 grid ((d.ow + L2Shape<TH, 1>::TW - 1) / L2Shape<TH, 1>::TW, (d.oh + TH - 1) / TH, n);
  kern <<<grid, NT, L2Shape<TH, 1>::SMEM, stream>>> (d, st.dev, v2.dev, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

inline int launch_lanczos2_v2 (const VcsDev & d, const Lanczos2State & st, const Lanczos2V2State & v2, const VcsBatch & batch, int n,
    cudaStream_t stream, bool planar_out = false)
{
  if (planar_out) {                               // RGBP (sel of RGBx) / BGRP (sel of BGRx)
    const bool bgr = d.sel == 0x0123u;
    if (d.planar)
      return bgr ? launch_lanczos2_v2_sel<0x0123, true, false, true> (d, st, v2, batch, n, stream)
                 : launch_lanczos2_v2_sel<0x0321, true, false, true> (d, st, v2, batch, n, stream);
    return bgr ? launch_lanczos2_v2_sel<0x0123, false, false, true> (d, st, v2, batch, n, stream)
               : launch_lanczos2_v2_sel<0x0321, false, false, true> (d, st, v2, batch, n, stream);
  }
  if (d.yuv_out)                                  // the cross-family chain's first launch: scaled {255, Y, U, V} pixels, no matrix
    return d.planar ? launch_lanczos2_v2_sel<-1, true, true> (d, st, v2, batch, n, stream)
                    : launch_lanczos2_v2_sel<-1, false, true> (d, st, v2, batch, n, stream);
  if (d.planar) {                                 // I420 / YV12 input
    switch (d.sel) {
      case 0x0123u: return launch_lanczos2_v2_sel<0x0123, true> (d, st, v2, batch, n, stream);
      case 0x0321u: return launch_lanczos2_v2_sel<0x0321, true> (d, st, v2, batch, n, stream);
      default: return launch_lanczos2_v2_sel<-1, true> (d, st, v2, batch, n, stream);
    }
  }
  switch (d.sel) {
    case 0x0123u: return launch_lanczos2_v2_sel<0x0123> (d, st, v2, batch, n, stream);   // BGRA / BGRx
    case 0x0321u: return launch_lanczos2_v2_sel<0x0321> (d, st, v2, batch, n, stream);   // RGBA / RGBx
    default: return launch_lanczos2_v2_sel<-1> (d, st, v2, batch, n, stream);
  }
}

}  // namespace b200
