// gstreamer_b200/csrc/vcs_l2mma.cuh — experimental variant of the headline kernel (product code, sm_90a; opt-in).
//
// Same shape class and the same arithmetic as vcs_lanczos2_kernel (4:2:0 semi-planar -> packed RGB, exact 2:1 in both
// directions, 8-tap filters, h-cosited chroma, lines consumed in order), but the two FIR passes run on the integer
// tensor path: a 2:1 8-tap FIR over u8 samples with s8 taps and exact s32 accumulation IS a banded matrix product, and
// IMMA.16832.U8.S8 (mma.sync.m16n8k32) computes 128 FIR outputs per warp instruction where the SIMT kernel spends
// 2-3 IDP.4A plus alignment work per output.  The measured limiter of the SIMT kernel is instruction issue
// (DESIGN.md 4.2), which is what this variant attacks; it has not been timed on the H100 and is
// selected only by b200_vcs_set_kernel_variant (h, 6).
//
//  stage A  a thread prepares 4 lines x 8 input pixels: Y copied, chroma de-interleaved, co-sited h up-sampling and the
//           (3a+b+2)>>2 line pairs as packed byte averages (the code of vcs_lanczos2_kernel's H phase), written as planar
//           Y / U / V byte rows of the tile's input region to shared memory.  Indices are clamped at the frame borders;
//           samples outside the frame are never referenced by a tap (the reference folds edge taps), so any byte will do.
//  H        a warp owns 8 output columns for all 64 staged lines: A = 16 line-groups x a 32-byte column window
//           (LDS.64 per fragment half; MMA i of 4 takes line i of every group, so a thread ends up with 4 consecutive
//           lines of its two groups and packs them into one word), B = the tap band of those 8 columns from a host table
//           (edge columns simply have other taps there), C preset to the rounding constant (128: the tables carry the taps times 4, so that the rounded, saturated result is
//           byte 1 of a saturating 16-bit pack - no shifts).  Result words
//           [line-group][column] = 4 lines of one column, as in the SIMT kernel.
//  V        a warp owns 16 columns x 8 output rows: A = columns x 32 staged lines (the words above), B = the vertical tap
//           band, C = 32; epilogue per pixel = the SIMT kernel's: saturate, mulhi matrix, byte order, store.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <vector>

#include "common.h"
#include "vcs_device.h"
#include "vcs_plan.h"
#include "vcs_lanczos2.cuh"      // packed-byte averages, saturating packs, sign-splat permutes

namespace b200 {

constexpr int LM_TW = 64, LM_TH = 24;          // output tile
constexpr int LM_NG = 16;                       // line groups of 4 staged lines (2*TH+6 = 54 lines -> 14 used; the MMA's M is 16)
constexpr int LM_UNITS = (2 * LM_TW + 16) / 8;  // 8-pixel units per staged line (8 halo pixels each side)
// staged input bytes: [channel][line of its group i][group pair g][word column w][group g | group g+8], i.e. the two
// line groups the MMA's rows g and g+8 stand for are interleaved word by word, so that ONE LDS.128 at word column 4j+2t
// returns a0 (row g, window bytes 8t..8t+3), a1 (row g+8, same bytes), a2 (row g, bytes 8t+4..), a3 (row g+8) - the
// fragment in the register order the instruction wants (IMMA overwrites its A registers with D: a fresh load per MMA is
// what it takes anyway)
constexpr int LM_WP = 40;                       // word columns per staged row (>= 36; row pitch 320 B = 64 mod 128: conflict-free)
constexpr int LM_PLANE = 4 * 8 * LM_WP * 8;     // bytes per staged channel
constexpr int LM_HP = LM_TW + 8;                // pitch of the h-scaled words (72: rows 8 banks apart)
constexpr int LM_SMEM = 3 * LM_PLANE + 3 * LM_NG * LM_HP * 4;

struct L2mmaDev {
  const uint2 *bh;               // [ow/8][32 lanes]: B fragment (b0, b1) of each group of 8 output columns
  const uint2 *bv;               // [oh/8][32 lanes]
  // per group: 1 = the table carries the taps times 4 (accumulator preset 128, result = byte 1 of a saturating 16-bit
  // pack, no shifts); 0 = plain taps (preset 32, shift by 6) - groups at a frame border, whose folded taps reach 32
  const uint8_t *h4, *v4;
};

// D = A(16x32 u8, row) * B(32x8 s8, col) + c  (mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32); all 4 accumulators
// start at the same constant
__device__ __forceinline__ void mma_u8s8 (int (&d)[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0,
    unsigned b1, const int (&c)[4])
{
#ifdef B200_CUDA_EMU
  b200emu::warp_mma_u8s8 (d, a0, a1, a2, a3, b0, b1, c);
#else
  asm volatile ("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
      : "=r" (d[0]), "=r" (d[1]), "=r" (d[2]), "=r" (d[3])
      : "r" (a0), "r" (a1), "r" (a2), "r" (a3), "r" (b0), "r" (b1), "r" (c[0]), "r" (c[1]), "r" (c[2]), "r" (c[3]));
#endif
}

// the same product with the operand types swapped: A s8 (taps), B u8 (pixels)
__device__ __forceinline__ void mma_s8u8 (int (&d)[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0,
    unsigned b1, const int (&c)[4])
{
#ifdef B200_CUDA_EMU
  b200emu::warp_mma_s8u8 (d, a0, a1, a2, a3, b0, b1, c);
#else
  asm volatile ("mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
      : "=r" (d[0]), "=r" (d[1]), "=r" (d[2]), "=r" (d[3])
      : "r" (a0), "r" (a1), "r" (a2), "r" (a3), "r" (b0), "r" (b1), "r" (c[0]), "r" (c[1]), "r" (c[2]), "r" (c[3]));
#endif
}

// EDGE = the tile touches a frame border: line / chroma-row / column indices are clamped and the "no chroma sample to the
// right" case exists; interior tiles run the instantiation without any of it (same split as vcs_lanczos2_kernel).
template <bool EDGE>
__device__ __forceinline__ void l2mma_tile (const VcsDev & P, const L2mmaDev & L, const uint8_t *__restrict__ in,
    uint8_t *__restrict__ out, uint8_t *smem, int x0, int oy0)
{
  uint8_t *S = smem;                                             // [3][4][8][LM_WP][2] words, see LM_WP
  unsigned *HS = (unsigned *) (smem + 3 * LM_PLANE);             // [3][LM_NG][LM_HP] words: 4 lines of one h-scaled column
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const uint8_t *__restrict__ plane_y = in + P.off_y;
  const uint8_t *__restrict__ plane_c = in + P.off_c;
  const int R0 = 2 * oy0 - 3;                                    // first staged line; R0 % 4 == 1
  const int crows = P.ih >> 1;
  const unsigned selU = P.u_index ? 0x7531u : 0x6420u, selV = P.u_index ? 0x6420u : 0x7531u;

  // ---------------------------------------------------------------- stage A: Y and full-resolution chroma of the region
  for (int item = tid; item < (LM_NG - 2) * LM_UNITS; item += L2_THREADS) {
    const int lg = item / LM_UNITS, u = item - lg * LM_UNITS;
    const int xraw = 2 * x0 - 8 + 8 * u;
    const int xb = EDGE ? min (max (xraw, 0), P.iw - 8) : xraw;  // byte column of the unit's 8 input pixels
    const bool right_edge = EDGE && xb + 8 >= P.iw;              // no chroma sample to the right
    const int y0 = R0 + 4 * lg;                                  // lines y0..y0+3, y0 % 4 == 1
    const int m2 = (y0 - 1) >> 1;                                // chroma rows m2, m2+1, m2+2
    unsigned ulo[3], uhi[3], vlo[3], vhi[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const int cr = EDGE ? min (max (m2 + k, 0), crows - 1) : m2 + k;
      const uint8_t *row = plane_c + (unsigned) cr * (unsigned) P.stride_c + (unsigned) xb;
      const uint2 c = __ldg ((const uint2 *) row);
      const unsigned ue = __byte_perm (c.x, c.y, selU), ve = __byte_perm (c.x, c.y, selV);
      unsigned un, vn;
      if (right_edge) {
        un = __byte_perm (ue, ue, 0x3321);
        vn = __byte_perm (ve, ve, 0x3321);
      } else {                                                   // the first sample pair of the next unit
        const unsigned nx = __ldg ((const unsigned short *) (row + 8));
        un = __byte_perm (ue, nx, P.u_index ? 0x5321 : 0x4321);
        vn = __byte_perm (ve, nx, P.u_index ? 0x4321 : 0x5321);
      }
      const unsigned uo = avg_ceil4 (ue, un), vo = avg_ceil4 (ve, vn);        // video-chroma.c:687-699
      ulo[k] = __byte_perm (ue, uo, 0x5140); uhi[k] = __byte_perm (ue, uo, 0x7362);
      vlo[k] = __byte_perm (ve, vo, 0x5140); vhi[k] = __byte_perm (ve, vo, 0x7362);
    }
    // vertical pairs (4m+1,4m+2) on rows (a,b) and (4m+3,4m+4) on rows (b,c): (3x+y+2)>>2 == avg_ceil (x, avg_floor (x,y))
    uint2 U[4], V[4];
    {
      unsigned f;
      f = avg_floor4 (ulo[0], ulo[1]); U[0].x = avg_ceil4 (ulo[0], f); U[1].x = avg_ceil4 (ulo[1], f);
      f = avg_floor4 (uhi[0], uhi[1]); U[0].y = avg_ceil4 (uhi[0], f); U[1].y = avg_ceil4 (uhi[1], f);
      f = avg_floor4 (ulo[1], ulo[2]); U[2].x = avg_ceil4 (ulo[1], f); U[3].x = avg_ceil4 (ulo[2], f);
      f = avg_floor4 (uhi[1], uhi[2]); U[2].y = avg_ceil4 (uhi[1], f); U[3].y = avg_ceil4 (uhi[2], f);
      f = avg_floor4 (vlo[0], vlo[1]); V[0].x = avg_ceil4 (vlo[0], f); V[1].x = avg_ceil4 (vlo[1], f);
      f = avg_floor4 (vhi[0], vhi[1]); V[0].y = avg_ceil4 (vhi[0], f); V[1].y = avg_ceil4 (vhi[1], f);
      f = avg_floor4 (vlo[1], vlo[2]); V[2].x = avg_ceil4 (vlo[1], f); V[3].x = avg_ceil4 (vlo[2], f);
      f = avg_floor4 (vhi[1], vhi[2]); V[2].y = avg_ceil4 (vhi[1], f); V[3].y = avg_ceil4 (vhi[2], f);
    }
    unsigned *d = (unsigned *) S + ((lg & 7) * LM_WP + 2 * u) * 2 + (lg >> 3);   // word (line 0, pair lg&7, column 2u, half lg>>3)
    const uint8_t *py = plane_y + (unsigned) xb;
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int y = EDGE ? min (max (y0 + r, 0), P.ih - 1) : y0 + r;
      const uint2 yy = __ldg ((const uint2 *) (py + (unsigned) y * (unsigned) P.stride_y));
      unsigned *dr = d + r * 8 * LM_WP * 2;
      dr[0] = yy.x; dr[2] = yy.y;
      dr[LM_PLANE / 4] = U[r].x; dr[LM_PLANE / 4 + 2] = U[r].y;
      dr[2 * (LM_PLANE / 4)] = V[r].x; dr[2 * (LM_PLANE / 4) + 2] = V[r].y;
    }
  }
  __syncthreads ();

  // ---------------------------------------------------------------- H phase: warp = 8 output columns, all staged lines
  for (int j = warp; j < LM_TW / 8; j += L2_THREADS / 32) {
    if (x0 + 8 * j >= P.ow) continue;                              // partial last tile: no such columns (warp-uniform)
    const uint2 B = __ldg (L.bh + ((x0 >> 3) + j) * 32 + lane);
    const bool x4 = __ldg (L.h4 + (x0 >> 3) + j) != 0;              // warp-uniform
    const int ci = x4 ? 128 : 32;
    const int c_init[4] = {ci, ci, ci, ci};
    const uint4 *frag = (const uint4 *) S + (g * LM_WP + 4 * j + 2 * t) / 2;      // 16 bytes: a0, a1, a2, a3 of line 0
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
      int d[4][4];                                               // [line of the group][fragment element]
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const uint4 a = frag[(ch * LM_PLANE + i * 8 * LM_WP * 8) / 16];
        mma_u8s8 (d[i], a.x, a.y, a.z, a.w, B.x, B.y, c_init);
      }
      // (acc+32)>>6 saturated to u8 (video-orc.orc:2474-2481); byte i of a word = line i of the group
      uint2 wlo, whi;
      if (x4) {                  // = byte 1 of sat_u16 (4 acc + 128)
        wlo.x = __byte_perm (pack_sat_u16x2 (d[1][0], d[0][0]), pack_sat_u16x2 (d[3][0], d[2][0]), 0x7531);
        wlo.y = __byte_perm (pack_sat_u16x2 (d[1][1], d[0][1]), pack_sat_u16x2 (d[3][1], d[2][1]), 0x7531);
        whi.x = __byte_perm (pack_sat_u16x2 (d[1][2], d[0][2]), pack_sat_u16x2 (d[3][2], d[2][2]), 0x7531);
        whi.y = __byte_perm (pack_sat_u16x2 (d[1][3], d[0][3]), pack_sat_u16x2 (d[3][3], d[2][3]), 0x7531);
      } else {
        wlo.x = pack_sat2 (sra6 (d[1][0]), sra6 (d[0][0]), pack_sat2 (sra6 (d[3][0]), sra6 (d[2][0]), 0u));
        wlo.y = pack_sat2 (sra6 (d[1][1]), sra6 (d[0][1]), pack_sat2 (sra6 (d[3][1]), sra6 (d[2][1]), 0u));
        whi.x = pack_sat2 (sra6 (d[1][2]), sra6 (d[0][2]), pack_sat2 (sra6 (d[3][2]), sra6 (d[2][2]), 0u));
        whi.y = pack_sat2 (sra6 (d[1][3]), sra6 (d[0][3]), pack_sat2 (sra6 (d[3][3]), sra6 (d[2][3]), 0u));
      }
      unsigned *hs = HS + ch * LM_NG * LM_HP + 8 * j + 2 * t + g * LM_HP;
      *(uint2 *) hs = wlo;
      *(uint2 *) (hs + 8 * LM_HP) = whi;
    }
  }
  __syncthreads ();

  // ---------------------------------------------------------------- V phase: warp = 16 columns x 8 output rows
  for (int item = warp; item < (LM_TW / 16) * (LM_TH / 8); item += L2_THREADS / 32) {
    const int q = item / (LM_TW / 16), c0 = (item - q * (LM_TW / 16)) * 16;
    const int oyq = oy0 + 8 * q;
    if (oyq >= P.oh) continue;                                   // warp-uniform
    const uint2 B = __ldg (L.bv + (oyq >> 3) * 32 + lane);
    const bool x4 = __ldg (L.v4 + (oyq >> 3)) != 0;                 // warp-uniform
    const int ci = x4 ? 128 : 32;
    const int c_init[4] = {ci, ci, ci, ci};
    int d[3][4];
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
      const unsigned *hs = HS + ch * LM_NG * LM_HP + c0 + g + (4 * q + t) * LM_HP;
      mma_u8s8 (d[ch], hs[0], hs[8], hs[4 * LM_HP], hs[4 * LM_HP + 8], B.x, B.y, c_init);
    }
    uint8_t *orow = out + P.off_out + (unsigned) (oyq + 2 * t) * (unsigned) P.stride_out + (unsigned) (x0 + c0 + g) * 4u;
#pragma unroll
    for (int e = 0; e < 4; e++) {
      const int ox = x0 + c0 + g + 8 * (e >> 1), oy = oyq + 2 * t + (e & 1);
      if (ox >= P.ow || oy >= P.oh) continue;
      // saturate the three channels at once, bias by 128 and sign-splat each byte to s16 (video-orc.orc:1634-1688)
      unsigned yuv = x4 ? __byte_perm (pack_sat_u16x2 (d[1][e], d[0][e]), pack_sat_u16x2 (0, d[2][e]), 0x7531)
          : pack_sat2 (d[1][e] >> 6, d[0][e] >> 6, pack_sat2 (0, d[2][e] >> 6, 0u));
      yuv ^= 0x00808080u;
      const int wy = prmt_s (yuv, 0x8800u), wu = prmt_s (yuv, 0x9911u), wv = prmt_s (yuv, 0xaa22u);
      const int ty = ((wy * P.p1) >> 16) + 128;
      const int r = ty + ((wv * P.p2) >> 16);
      const int b = ty + ((wu * P.p3) >> 16);
      const int gg = ty + ((wu * P.p4) >> 16) + ((wv * P.p5) >> 16);
      const unsigned argb = pack_sat2 (r, 255, pack_sat2 (b, gg, 0u));
      *(unsigned *) (orow + (e & 1) * P.stride_out + (e >> 1) * 32) = __byte_perm (argb, 0, P.sel);
    }
  }
}

__global__ void __launch_bounds__ (L2_THREADS, 3)
vcs_l2mma_kernel (const VcsDev P, const L2mmaDev L, const VcsBatch frames)
{
  extern __shared__ __align__ (16) uint8_t smem[];
  const int x0 = blockIdx.x * LM_TW, oy0 = blockIdx.y * LM_TH;
  // staged region: lines 2*oy0-3 .. +55 (groups 14, 15 are never written: no tap references them), columns 2*x0-8 .. +143
  const bool edge = 2 * oy0 - 3 < 0 || 2 * oy0 - 3 + 4 * (LM_NG - 2) > P.ih || x0 == 0 || 2 * x0 - 8 + 8 * LM_UNITS + 8 > P.iw;
  if (edge) l2mma_tile<true> (P, L, frames.in[blockIdx.z], frames.out[blockIdx.z], smem, x0, oy0);
  else l2mma_tile<false> (P, L, frames.in[blockIdx.z], frames.out[blockIdx.z], smem, x0, oy0);
}

// ------------------------------------------------------------------------------------ host side
struct L2mmaTables {
  std::vector<uint32_t> bh, bv;        // [groups][32 lanes][2]
  std::vector<uint8_t> h4, v4;         // [groups]: taps stored times 4
  bool ok = false;
};

// B fragments of one axis: group T covers outputs 8T..8T+7 and the 32 input samples starting at 16T - bias.
// Fragment element k of lane (g, t), register r, byte b: k = 16r + 4t + b, n = g; the sample k stands for is
// window[k] (h: the 8-byte interleave that lets a thread fetch its two fragment registers with one LDS.64).
inline bool pack_axis_l2mma (const AxisPlan & a, int bias, bool interleave8, std::vector<uint32_t> * tab,
    std::vector<uint8_t> * times4)
{
  if (a.mode != PASS_NTAP || a.n_taps != 8 || a.in_size != 2 * a.out_size || (a.out_size & 7)) return false;
  const int groups = a.out_size / 8;
  tab->assign ((size_t) groups * 64, 0);
  times4->assign (groups, 1);
  for (int T = 0; T < groups; T++) {
    for (int j = 8 * T; j < 8 * T + 8; j++)             // taps times 4 must fit s8: not where folded edge taps reach 32
      for (int k = 0; k < 8; k++)
        if (4 * a.coef[(size_t) j * 8 + k] < -128 || 4 * a.coef[(size_t) j * 8 + k] > 127) (*times4)[T] = 0;
    const int scale = (*times4)[T] ? 4 : 1;
    for (int n = 0; n < 8; n++) {
      const int j = 8 * T + n;
      int8_t col[32] = {0};
      int mag = 0;
      for (int k = 0; k < 8; k++) {
        const int tap = a.coef[(size_t) j * 8 + k];
        mag += abs (tap);
        if (tap == 0) continue;
        const int pos = (int) a.offset[j] + k - (16 * T - bias);               // window sample index
        if (pos < 0 || pos >= 32 || tap < -128 || tap > 127) return false;
        col[pos] = (int8_t) (scale * tap);
      }
      if (255 * mag + 32 > 32767) return false;        // must stay inside the reference's 16-bit accumulator (unscaled taps)
      for (int k = 0; k < 32; k++) {
        // which window sample does fragment element k hold?
        const int w = interleave8 ? 8 * ((k & 15) >> 2) + (k & 3) + ((k >> 4) ? 4 : 0) : k;
        const int lane = n * 4 + ((k & 15) >> 2), reg = k >> 4, byte = k & 3;
        (*tab)[(size_t) T * 64 + lane * 2 + reg] |= (uint32_t) (uint8_t) col[w] << (8 * byte);
      }
    }
  }
  return true;
}

inline L2mmaTables build_l2mma_tables (const VcsPlan & p)
{
  L2mmaTables t;
  if (p.yuv_out || p.rgb_in || p.planes_mode) return t;
  if (!p.h_first || p.matrix_first || !p.h_cosited || !p.v_pairs || p.planar || p.chroma_nearest) return t;
  if ((p.in.stride[0] & 7) || (p.in.stride[1] & 7) || (p.in.offset[0] & 7) || (p.in.offset[1] & 7)) return t;
  if ((p.in.width & 7) || (p.in.height & 1) || p.in.width < 8) return t;
  if ((p.out.stride[0] & 3) || (p.out.offset[0] & 3)) return t;
  if (!standard_pairing (p)) return t;
  if (!alpha_stays_opaque (p.h) || !alpha_stays_opaque (p.v)) return t;     // alpha stays 255 through both passes
  if (!pack_axis_l2mma (p.h, 8, true, &t.bh, &t.h4)) return t;     // staged columns start 8 pixels left of the tile
  if (!pack_axis_l2mma (p.v, 3, false, &t.bv, &t.v4)) return t;    // staged lines start at 2*oy0 - 3
  t.ok = true;
  return t;
}

struct L2mmaState {
  uint32_t *d_bh = nullptr, *d_bv = nullptr;
  uint8_t *d_h4 = nullptr, *d_v4 = nullptr;
  L2mmaDev dev;
  bool ready = false;
};

inline int prepare_l2mma (const L2mmaTables & t, L2mmaState * st)
{
  int rc;
  if ((rc = upload (&st->d_bh, t.bh.data (), t.bh.size ())) != B200_OK) return rc;
  if ((rc = upload (&st->d_bv, t.bv.data (), t.bv.size ())) != B200_OK) return rc;
  if ((rc = upload (&st->d_h4, t.h4.data (), t.h4.size ())) != B200_OK) return rc;
  if ((rc = upload (&st->d_v4, t.v4.data (), t.v4.size ())) != B200_OK) return rc;
  st->dev.bh = (const uint2 *) st->d_bh;
  st->dev.bv = (const uint2 *) st->d_bv;
  st->dev.h4 = st->d_h4; st->dev.v4 = st->d_v4;
  B200_CUDA_TRY (cudaFuncSetAttribute (vcs_l2mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LM_SMEM));
  st->ready = true;
  return B200_OK;
}

inline int launch_l2mma (const VcsDev & d, const L2mmaState & st, const VcsBatch & batch, int n, cudaStream_t stream)
{
  dim3 grid ((d.ow + LM_TW - 1) / LM_TW, (d.oh + LM_TH - 1) / LM_TH, n);
  vcs_l2mma_kernel <<<grid, L2_THREADS, LM_SMEM, stream>>> (d, st.dev, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
