// gstreamer_b200/csrc/vcs_lanczos2.cuh — specialised fused kernel for the headline shape class
// (product code, sm_90a): 4:2:0 semi-planar -> packed RGB, exact 2:1 reduction in both
// directions with the 8-tap filters the reference derives for it (lanczos and every other
// 8-tap/2:1 method), h-cosited chroma, all input lines consumed in order.
//
// Same arithmetic as vcs_generic_kernel (and therefore as the reference chain
// unpack -> chroma up h,v -> h scale -> v scale -> AYUV->ARGB -> pack, see vcs_kernels.cuh),
// organised for instruction count instead of generality:
//
//  * byte-SIMD everywhere: 4 pixels per 32-bit register; chroma up-sampling is done with
//    packed byte averages ((a+b+1)>>1 and (3a+b+2)>>2 == avg_ceil(a, avg_floor(a,b))), the FIRs
//    with IDP.4A.U8.S8 on aligned words and zero-padded tap words (no funnel shifts)
//  * H phase: a warp owns 4 input lines x 128 input-aligned output columns straight from global
//    memory (LDG.64 per lane, halo words by warp shuffle, lanes 0/31 are halo providers), and
//    writes the h-scaled bytes TRANSPOSED (4 consecutive lines of one column per word) with one
//    STS.128 per channel
//  * V phase: a thread owns 4 output rows of one column: 4 LDS.32 per channel give the 16 lines
//    it needs, IDP.4A again, I2IP saturating packs, PRMT sign-splat for the mulhi matrix,
//    coalesced 4-byte stores
//  * the per-column / per-row tap words (12 registers each) come from host-built tables, so the
//    folded, non-uniform taps at the frame edges need no special code path.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <type_traits>
#include <vector>

#include "common.h"
#include "vcs_device.h"
#include "vcs_plan.h"

namespace b200 {

// tile shape: TH output rows x NWC warp-columns of 120 useful output columns (30 lanes x 4; lanes
// 0 and 31 only provide halo words).  A tile needs 2*TH + 6 input lines = NG groups of 4.
constexpr int L2_WCOLS = 120;
constexpr int L2_THREADS = 256;
template <int TH, int NWC> struct L2Shape {
  static constexpr int NG = (2 * TH + 6 + 3) / 4;
  static constexpr int TW = L2_WCOLS * NWC;
  static constexpr int TWP = 128 * NWC;       // smem columns incl. the halo lanes' slots
  static constexpr int SMEM = 3 * NG * TWP * 4;
};

struct Lanczos2Dev {
  const int4 *htab;                    // [ow/4][3] : 12 packed s8x4 tap words per 4-column group
  const int4 *vtab;                    // [oh/4][3]
  const short *hsum, *vsum;            // tap sums (alpha channel)
  int alpha_opaque;                    // every tap sum >= 64: alpha is 255 everywhere
  // X4 instantiation (opt-in): the same tables with every tap times 4.  With the accumulator preset to 128 the rounded,
  // saturated FIR output is byte 1 of a saturating 16-bit pack of 4 acc + 128 - one I2IP per two outputs and one PRMT
  // per four instead of a shift per output.  Folded taps at the frame borders reach 32 (x4 = 128 does not fit s8): edge
  // tiles keep the plain tables in the H phase, and v4[row group] says which row groups may use vtab4.
  const int4 *htab4, *vtab4;
  const uint8_t *v4;
};

// ---- packed byte helpers -----------------------------------------------------------------
// ((a ^ b) & 0xfefefefe) as ONE LOP3 (lut 0x28); written in PTX because the compiler otherwise
// re-associates the mask behind the shift and spends a second LOP3 on it
__device__ __forceinline__ unsigned xor_and_fe (unsigned a, unsigned b)
{
#ifdef B200_CUDA_EMU               // host build of the kernel sources for tests/cudaemu: same function, plain C
  return (a ^ b) & 0xfefefefeu;
#else
  unsigned d;
  asm ("lop3.b32 %0, %1, %2, 0xfefefefe, 0x28;" : "=r" (d) : "r" (a), "r" (b));
  return d;
#endif
}
__device__ __forceinline__ unsigned avg_floor4 (unsigned a, unsigned b)
{
  return (a & b) + (xor_and_fe (a, b) >> 1);
}
__device__ __forceinline__ unsigned avg_ceil4 (unsigned a, unsigned b)
{
  return (a | b) - (xor_and_fe (a, b) >> 1);
}
__device__ __forceinline__ int dp4a_u8s8 (unsigned px, int taps, int acc)
{
#ifdef B200_CUDA_EMU
  for (int i = 0; i < 4; i++) acc += (int) ((px >> (8 * i)) & 0xff) * (int) (int8_t) ((unsigned) taps >> (8 * i));
  return acc;
#else
  int d;
  asm ("dp4a.u32.s32 %0, %1, %2, %3;" : "=r" (d) : "r" (px), "r" (taps), "r" (acc));
  return d;
#endif
}
__device__ __forceinline__ int prmt_s (unsigned a, unsigned sel)      // prmt.b32: selector msb replicates the sign
{
#ifdef B200_CUDA_EMU
  return (int) __byte_perm (a, 0, sel);
#else
  int d;
  asm ("prmt.b32 %0, %1, 0, %2;" : "=r" (d) : "r" (a), "r" (sel));
  return d;
#endif
}
// acc >> 6 (arithmetic).  SHF runs at half rate on the ALU pipe; IMAD.HI would be a quarter-rate
// alternative, so the plain shift stays.
__device__ __forceinline__ int sra6 (int acc) { return acc >> 6; }
// d = { c[15:0], sat_u8(a), sat_u8(b) }  (b in the lowest byte)
__device__ __forceinline__ unsigned pack_sat2 (int a, int b, unsigned c)
{
#ifdef B200_CUDA_EMU
  return (c << 16) | ((unsigned) min (max (a, 0), 255) << 8) | (unsigned) min (max (b, 0), 255);
#else
  unsigned d;
  asm ("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r" (d) : "r" (a), "r" (b), "r" (c));
  return d;
#endif
}

// d = { sat_u16(a), sat_u16(b) }  (b in the low half).  With taps scaled by 4 and the accumulator preset to 128 the
// rounded, saturated FIR output (acc + 32) >> 6 clamped to [0, 255] is byte 1 of sat_u16 (4 acc + 128): no shift needed
__device__ __forceinline__ unsigned pack_sat_u16x2 (int a, int b)
{
#ifdef B200_CUDA_EMU
  return ((unsigned) min (max (a, 0), 65535) << 16) | (unsigned) min (max (b, 0), 65535);
#else
  unsigned d;
  asm ("cvt.pack.sat.u16.s32 %0, %1, %2;" : "=r" (d) : "r" (a), "r" (b));
  return d;
#endif
}

// 4 outputs from 16 aligned bytes w0..w3: outputs 0,1 read words 0..2, outputs 2,3 words 1..3
#define L2_FIR4(o0, o1, o2, o3, w0, w1, w2, w3, T, INIT)                                       \
  do {                                                                                         \
    o0 = dp4a_u8s8 (w2, T[0].z, dp4a_u8s8 (w1, T[0].y, dp4a_u8s8 (w0, T[0].x, INIT)));         \
    o1 = dp4a_u8s8 (w2, T[1].y, dp4a_u8s8 (w1, T[1].x, dp4a_u8s8 (w0, T[0].w, INIT)));         \
    o2 = dp4a_u8s8 (w3, T[2].x, dp4a_u8s8 (w2, T[1].w, dp4a_u8s8 (w1, T[1].z, INIT)));         \
    o3 = dp4a_u8s8 (w3, T[2].w, dp4a_u8s8 (w2, T[2].z, dp4a_u8s8 (w1, T[2].y, INIT)));         \
  } while (0)

template <bool ALPHA_OPAQUE, int MINB, int TH, int NWC, bool X4 = false>
__global__ void __launch_bounds__ (L2_THREADS, MINB)
vcs_lanczos2_kernel (const VcsDev P, const Lanczos2Dev L, const VcsBatch frames)
{
  constexpr int L2_TH = TH, L2_NWC = NWC, L2_NG = L2Shape<TH, NWC>::NG, L2_TW = L2Shape<TH, NWC>::TW,
      L2_TWP = L2Shape<TH, NWC>::TWP;
  extern __shared__ __align__ (16) unsigned hs[];                // [3][L2_NG][L2_TWP] words
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync (0xffffffffu, (int) (threadIdx.x >> 5), 0);   // warp-uniform for the compiler
  const uint8_t *__restrict__ in = frames.in[blockIdx.z];
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const uint8_t *__restrict__ plane_y = in + P.off_y;
  const uint8_t *__restrict__ plane_c = in + P.off_c;
  const int x0 = blockIdx.x * L2_TW, oy0 = blockIdx.y * L2_TH;
  const int R0 = 2 * oy0 - 3;                                    // first input line of the tile
  const int crows = P.ih >> 1;
  const unsigned selU = P.u_index ? 0x7531u : 0x6420u, selV = P.u_index ? 0x6420u : 0x7531u;

  // ---------------------------------------------------------------- H phase
  // Tiles that touch no frame border skip every clamp (line / chroma-row / column indices and the
  // "no chroma sample to the right" fix-up): warp-uniform choice between two instantiations.
  const bool edge_tile = R0 < 0 || R0 + 4 * L2_NG > P.ih || x0 == 0 || x0 + L2_TW + 4 >= P.ow;
  auto h_phase = [&] (auto edge_tag) {
    constexpr bool EDGE = decltype (edge_tag)::value;
    constexpr bool H4 = X4 && !EDGE;                             // interior tiles only: no folded taps there
    constexpr int HINIT = H4 ? 128 : 32;
    const int4 *__restrict__ htab = H4 ? L.htab4 : L.htab;
  for (int item = warp; item < L2_NG * L2_NWC; item += L2_THREADS / 32) {
    const int g = item / L2_NWC, wc = item - g * L2_NWC;
    const int col0 = x0 + wc * L2_WCOLS + (lane - 1) * 4;        // first of this lane's 4 output columns
    int4 T[3];
    {
      const int grp = EDGE ? min (max (col0 >> 2, 0), (P.ow >> 2) - 1) : (col0 >> 2);
      T[0] = __ldg (htab + grp * 3 + 0);
      T[1] = __ldg (htab + grp * 3 + 1);
      T[2] = __ldg (htab + grp * 3 + 2);
    }
    const int xb = EDGE ? min (max (2 * col0, 0), P.iw - 8) : 2 * col0;   // byte column of the lane's 8 input pixels
    const bool right_edge = EDGE && 2 * col0 + 8 >= P.iw;        // no chroma sample to the right
    const int y0 = R0 + 4 * g;                                   // lines y0..y0+3, y0 % 4 == 1
    const int m2 = (y0 - 1) >> 1;                                // chroma rows m2, m2+1, m2+2

    // chroma: three rows, de-interleave, cosited h up-sample (video-chroma.c:687-699)
    unsigned ulo[3], uhi[3], vlo[3], vhi[3];
    // interior tiles: one 64-bit address per plane and item, then row-to-row steps (the per-row index form costs a
    // 64-bit multiply-add per load)
    const uint8_t *pc = plane_c + (ptrdiff_t) m2 * P.stride_c + xb;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const int cr = EDGE ? min (max (m2 + k, 0), crows - 1) : m2 + k;
      const uint2 c = __ldg ((const uint2 *) (EDGE ? plane_c + (size_t) cr * P.stride_c + xb : pc));
      pc += P.stride_c;
      const unsigned ue = __byte_perm (c.x, c.y, selU), ve = __byte_perm (c.x, c.y, selV);
      unsigned un = __shfl_down_sync (0xffffffffu, ue, 1), vn = __shfl_down_sync (0xffffffffu, ve, 1);
      if (EDGE) {
        un = right_edge ? __byte_perm (ue, ue, 0x3321) : __byte_perm (ue, un, 0x4321);
        vn = right_edge ? __byte_perm (ve, ve, 0x3321) : __byte_perm (ve, vn, 0x4321);
      } else {
        un = __byte_perm (ue, un, 0x4321);
        vn = __byte_perm (ve, vn, 0x4321);
      }
      const unsigned uo = avg_ceil4 (ue, un), vo = avg_ceil4 (ve, vn);
      ulo[k] = __byte_perm (ue, uo, 0x5140); uhi[k] = __byte_perm (ue, uo, 0x7362);
      vlo[k] = __byte_perm (ve, vo, 0x5140); vhi[k] = __byte_perm (ve, vo, 0x7362);
    }
    // vertical pairs (4m+1,4m+2) on rows (a,b) and (4m+3,4m+4) on rows (b,c):
    // (3x+y+2)>>2 == avg_ceil (x, avg_floor (x,y))   (video-orc.orc:2705-2735)
    unsigned U[4][2], V[4][2];
    {
      unsigned f;
      f = avg_floor4 (ulo[0], ulo[1]); U[0][0] = avg_ceil4 (ulo[0], f); U[1][0] = avg_ceil4 (ulo[1], f);
      f = avg_floor4 (uhi[0], uhi[1]); U[0][1] = avg_ceil4 (uhi[0], f); U[1][1] = avg_ceil4 (uhi[1], f);
      f = avg_floor4 (ulo[1], ulo[2]); U[2][0] = avg_ceil4 (ulo[1], f); U[3][0] = avg_ceil4 (ulo[2], f);
      f = avg_floor4 (uhi[1], uhi[2]); U[2][1] = avg_ceil4 (uhi[1], f); U[3][1] = avg_ceil4 (uhi[2], f);
      f = avg_floor4 (vlo[0], vlo[1]); V[0][0] = avg_ceil4 (vlo[0], f); V[1][0] = avg_ceil4 (vlo[1], f);
      f = avg_floor4 (vhi[0], vhi[1]); V[0][1] = avg_ceil4 (vhi[0], f); V[1][1] = avg_ceil4 (vhi[1], f);
      f = avg_floor4 (vlo[1], vlo[2]); V[2][0] = avg_ceil4 (vlo[1], f); V[3][0] = avg_ceil4 (vlo[2], f);
      f = avg_floor4 (vhi[1], vhi[2]); V[2][1] = avg_ceil4 (vhi[1], f); V[3][1] = avg_ceil4 (vhi[2], f);
    }

    // (acc+32)>>6 saturated to u8 (video-orc.orc:2474-2481); four lines of a column go into
    // one word so that the V phase finds its 16 lines in 4 aligned words
#define L2_PACK4(A, c)                                                                         \
    (H4 ? __byte_perm (pack_sat_u16x2 (A[1][c], A[0][c]), pack_sat_u16x2 (A[3][c], A[2][c]), 0x7531)              \
        : pack_sat2 (sra6 (A[1][c]), sra6 (A[0][c]), pack_sat2 (sra6 (A[3][c]), sra6 (A[2][c]), 0u)))
#define L2_STORE(ch, A)                                                                        \
    do {                                                                                       \
      uint4 o;                                                                                 \
      o.x = L2_PACK4 (A, 0); o.y = L2_PACK4 (A, 1); o.z = L2_PACK4 (A, 2); o.w = L2_PACK4 (A, 3); \
      *(uint4 *) (hs + ((ch) * L2_NG + g) * L2_TWP + wc * 128 + lane * 4) = o;                 \
    } while (0)

    int acc[4][4];                                               // [line][column]
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const unsigned w0 = __shfl_up_sync (0xffffffffu, U[r][1], 1), w3 = __shfl_down_sync (0xffffffffu, U[r][0], 1);
      L2_FIR4 (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, U[r][0], U[r][1], w3, T, HINIT);
    }
    L2_STORE (1, acc);
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const unsigned w0 = __shfl_up_sync (0xffffffffu, V[r][1], 1), w3 = __shfl_down_sync (0xffffffffu, V[r][0], 1);
      L2_FIR4 (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, V[r][0], V[r][1], w3, T, HINIT);
    }
    L2_STORE (2, acc);
    const uint8_t *py = plane_y + (ptrdiff_t) y0 * P.stride_y + xb;
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int y = EDGE ? min (max (y0 + r, 0), P.ih - 1) : y0 + r;
      const uint2 yy = __ldg ((const uint2 *) (EDGE ? plane_y + (size_t) y * P.stride_y + xb : py));
      py += P.stride_y;
      const unsigned w0 = __shfl_up_sync (0xffffffffu, yy.y, 1), w3 = __shfl_down_sync (0xffffffffu, yy.x, 1);
      L2_FIR4 (acc[r][0], acc[r][1], acc[r][2], acc[r][3], w0, yy.x, yy.y, w3, T, HINIT);
    }
    L2_STORE (0, acc);
  }
  };
  if (edge_tile) h_phase (std::true_type {}); else h_phase (std::false_type {});
  __syncthreads ();

  // ---------------------------------------------------------------- V phase
  // a warp owns output rows oy0+4q .. +3 for all columns of the tile.  The taps-times-4 choice is warp-uniform and taken
  // as a BRANCH between two instantiations (as predicates both variants' packs would issue for every pixel); the column
  // loop is unrolled so that the four row pointers are formed once per row group and every store offset is an immediate.
  auto v_rows = [&] (auto v4_tag, int q) {
    constexpr bool V4 = decltype (v4_tag)::value;
    const int oy = oy0 + 4 * q;
    int4 T[3];
    const int4 *__restrict__ vtab = V4 ? L.vtab4 : L.vtab;
    constexpr int vinit = V4 ? 128 : 32;
    T[0] = __ldg (vtab + (oy >> 2) * 3 + 0);
    T[1] = __ldg (vtab + (oy >> 2) * 3 + 1);
    T[2] = __ldg (vtab + (oy >> 2) * 3 + 2);
    int vs[4] = {64, 64, 64, 64};
    if (!ALPHA_OPAQUE) {
#pragma unroll
      for (int i = 0; i < 4; i++) vs[i] = L.vsum[min (oy + i, P.oh - 1)];
    }
    uint8_t *rowp[4];                                            // oh % 4 == 0: all 4 rows exist
    rowp[0] = out + P.off_out + (size_t) oy * P.stride_out + (size_t) (x0 + lane) * 4u;
#pragma unroll
    for (int i = 1; i < 4; i++) rowp[i] = rowp[i - 1] + P.stride_out;
#pragma unroll
    for (int k = 0; k < (L2_TW + 31) / 32; k++) {
      const int c = lane + 32 * k;
      const int ox = x0 + c;
      if ((32 * k + 32 <= L2_TW || c < L2_TW) && ox < P.ow) {
        const int sc = c + 4 + (L2_NWC == 1 ? 0 : (c / L2_WCOLS) * (128 - L2_WCOLS));   // smem column of this output column
        int a[3][4];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
          const unsigned *p = hs + (ch * L2_NG + 2 * q) * L2_TWP + sc;
          const unsigned w0 = p[0], w1 = p[L2_TWP], w2 = p[2 * L2_TWP], w3 = p[3 * L2_TWP];
          L2_FIR4 (a[ch][0], a[ch][1], a[ch][2], a[ch][3], w0, w1, w2, w3, T, vinit);
        }
        int ah = 255;
        if (!ALPHA_OPAQUE) ah = fir_round_u8 ((int) (short) (255 * (int) L.hsum[ox]));
#pragma unroll
        for (int i = 0; i < 4; i++) {
          // saturate the three channels at once, bias by 128 and sign-splat each byte to s16
          unsigned yuv = V4 ? __byte_perm (pack_sat_u16x2 (a[1][i], a[0][i]), pack_sat_u16x2 (0, a[2][i]), 0x7531)
              : pack_sat2 (a[1][i] >> 6, a[0][i] >> 6, pack_sat2 (0, a[2][i] >> 6, 0u));
          yuv ^= 0x00808080u;
          const int wy = prmt_s (yuv, 0x8800u), wu = prmt_s (yuv, 0x9911u), wv = prmt_s (yuv, 0xaa22u);
          const int ty = ((wy * P.p1) >> 16) + 128;
          const int r = ty + ((wv * P.p2) >> 16);
          const int b = ty + ((wu * P.p3) >> 16);
          const int gg = ty + ((wu * P.p4) >> 16) + ((wv * P.p5) >> 16);
          int al = 255;
          if (!ALPHA_OPAQUE) al = fir_round_u8 ((int) (short) (ah * vs[i]));
          // ARGB bytes in one word, then the output format's byte order
          const unsigned argb = pack_sat2 (r, al, pack_sat2 (b, gg, 0u));
          *(unsigned *) (rowp[i] + 128 * k) = __byte_perm (argb, 0, P.sel);
        }
      }
    }
  };
  for (int q = warp; q < L2_TH / 4; q += L2_THREADS / 32) {
    const int oy = oy0 + 4 * q;
    if (oy < P.oh) {
      if (X4 && __ldg (L.v4 + (oy >> 2)) != 0) v_rows (std::true_type {}, q);     // this row group's taps fit s8 times 4
      else v_rows (std::false_type {}, q);
    }
  }
}

// ------------------------------------------------------------------------------------ host side
struct Lanczos2Tables {
  std::vector<int> htab, vtab;          // 12 words per group
  bool ok = false;
  bool alpha_opaque = false;
  // X4 instantiation: taps times 4 where they fit s8 (per 4-output group), see Lanczos2Dev
  std::vector<int> htab4, vtab4;
  std::vector<uint8_t> h4, v4;
  bool x4_ok = false;
};

// Place the taps of 4 consecutive outputs into their 16-sample aligned frame; outputs 0,1 may
// only touch samples 0..11 and outputs 2,3 samples 4..15.
inline bool pack_axis_lanczos2 (const AxisPlan & a, int frame_bias, std::vector<int> * tab, int scale = 1,
    std::vector<uint8_t> * fits = nullptr)
{
  if (a.mode != PASS_NTAP || a.n_taps != 8 || a.in_size != 2 * a.out_size || (a.out_size & 3))
    return false;
  const int groups = a.out_size / 4;
  tab->assign ((size_t) groups * 12, 0);
  if (fits) fits->assign (groups, 1);
  for (int gidx = 0; gidx < groups; gidx++) {
    const int base = 8 * gidx - frame_bias;
    if (fits)                                       // a scaled table: groups whose taps do not fit are left zero and flagged
      for (int j = 4 * gidx; j < 4 * gidx + 4; j++)
        for (int k = 0; k < 8; k++) {
          const int v = scale * a.coef[(size_t) j * 8 + k];
          if (v < -128 || v > 127) (*fits)[gidx] = 0;
        }
    if (fits && !(*fits)[gidx]) continue;
    for (int i = 0; i < 4; i++) {
      const int j = 4 * gidx + i;
      int8_t frame[16] = {0};
      for (int k = 0; k < 8; k++) {
        const int tap = a.coef[(size_t) j * 8 + k];
        if (tap == 0) continue;
        const int pos = (int) a.offset[j] + k - base;
        const int lo = i < 2 ? 0 : 4, hi = i < 2 ? 12 : 16;
        if (pos < lo || pos >= hi || scale * tap < -128 || scale * tap > 127) return false;
        frame[pos] = (int8_t) (scale * tap);
      }
      // 255 * sum(|taps|) + 32 must stay inside the reference's 16-bit accumulator
      int mag = 0;
      for (int k = 0; k < 8; k++) mag += abs ((int) a.coef[(size_t) j * 8 + k]);
      if (255 * mag + 32 > 32767) return false;
      const int first = i < 2 ? 0 : 1;
      for (int w = 0; w < 3; w++) {
        uint32_t word = 0;
        for (int b = 0; b < 4; b++) word |= (uint32_t) (uint8_t) frame[4 * (first + w) + b] << (8 * b);
        (*tab)[(size_t) gidx * 12 + i * 3 + w] = (int) word;
      }
    }
  }
  return true;
}

inline Lanczos2Tables build_lanczos2_tables (const VcsPlan & p)
{
  Lanczos2Tables t;
  if (!p.h_first || p.matrix_first || !p.h_cosited || !p.v_pairs || p.chroma_nearest) return t;
  if (p.planar) {                                 // I420 / YV12: only the second form of the kernel reads separate U and V planes (32-bit loads)
    if ((p.in.stride[0] & 7) || (p.in.offset[0] & 7)) return t;
    for (int k = 1; k <= 2; k++) if ((p.in.stride[k] & 3) || (p.in.offset[k] & 3) || p.in.stride[k] < (p.in.width >> 1)) return t;
  } else if ((p.in.stride[0] & 7) || (p.in.stride[1] & 7) || (p.in.offset[0] & 7) || (p.in.offset[1] & 7)) return t;
  if ((p.in.width & 7) || (p.in.height & 1)) return t;
  if (!standard_pairing (p)) return t;
  if (!pack_axis_lanczos2 (p.h, 4, &t.htab)) return t;
  if (!pack_axis_lanczos2 (p.v, 3, &t.vtab)) return t;
  t.alpha_opaque = alpha_stays_opaque (p.h) && alpha_stays_opaque (p.v);
  t.ok = true;
  // X4 tables: usable when every column group OUTSIDE the kernel's edge tiles (the first tile column and the tiles that
  // reach the right border: x0 == 0 || x0 + TW + 4 >= ow, TW = 120) fits; row groups are flagged one by one
  if (t.alpha_opaque && pack_axis_lanczos2 (p.h, 4, &t.htab4, 4, &t.h4) && pack_axis_lanczos2 (p.v, 3, &t.vtab4, 4, &t.v4)) {
    t.x4_ok = true;
    const int ow = p.out.width, TW = L2_WCOLS;
    for (size_t grp = 0; grp < t.h4.size (); grp++) {
      const int x0 = ((int) (4 * grp) / TW) * TW;
      const bool edge = x0 == 0 || x0 + TW + 4 >= ow;
      if (!edge && !t.h4[grp]) t.x4_ok = false;
    }
  }
  return t;
}

struct Lanczos2State {
  int4 *d_htab = nullptr, *d_vtab = nullptr;
  int4 *d_htab4 = nullptr, *d_vtab4 = nullptr;
  uint8_t *d_v4 = nullptr;
  Lanczos2Dev dev;
  int variant = 0;
  bool x4 = false;               // launch the X4 instantiation (whenever the tables allow it)
};

inline int prepare_lanczos2 (const Lanczos2Tables & t, const VcsDev & d, Lanczos2State * st)
{
  int rc;
  int *h = nullptr, *v = nullptr;
  if ((rc = upload (&h, t.htab.data (), t.htab.size ())) != B200_OK) return rc;
  if ((rc = upload (&v, t.vtab.data (), t.vtab.size ())) != B200_OK) return rc;
  st->d_htab = (int4 *) h; st->d_vtab = (int4 *) v;
  st->dev.htab = st->d_htab; st->dev.vtab = st->d_vtab;
  st->dev.hsum = d.h.sum; st->dev.vsum = d.v.sum;
  st->dev.alpha_opaque = t.alpha_opaque;
  st->dev.htab4 = st->dev.htab; st->dev.vtab4 = st->dev.vtab; st->dev.v4 = nullptr;
  const char *x4e = getenv ("B200_L2_X4");        // tuning knob: "0" keeps the plain tables
  if (t.x4_ok && !(x4e && x4e[0] == '0')) {      // the taps x 4 tables are the default; B200_L2_X4=0 selects the plain ones
    int *h4 = nullptr, *v4 = nullptr;
    if ((rc = upload (&h4, t.htab4.data (), t.htab4.size ())) != B200_OK) return rc;
    if ((rc = upload (&v4, t.vtab4.data (), t.vtab4.size ())) != B200_OK) return rc;
    if ((rc = upload (&st->d_v4, t.v4.data (), t.v4.size ())) != B200_OK) return rc;
    st->d_htab4 = (int4 *) h4; st->d_vtab4 = (int4 *) v4;
    st->dev.htab4 = st->d_htab4; st->dev.vtab4 = st->d_vtab4; st->dev.v4 = st->d_v4;
    st->x4 = true;
  }
  {
    const char *e = getenv ("B200_L2_VARIANT");      // tuning knob (0..3), see launch_lanczos2
    st->variant = e ? atoi (e) : 3;        // 120x60 tiles, 4 CTAs/SM
  }
  return B200_OK;
}

inline int launch_lanczos2 (const VcsDev & d, const Lanczos2State & st, const VcsBatch & batch, int n,
    cudaStream_t stream)
{
#define L2_LAUNCH(ALPHA, MINB, TH, NWC) L2_LAUNCH_X (ALPHA, MINB, TH, NWC, false)
#define L2_LAUNCH_X(ALPHA, MINB, TH, NWC, X4)                                                  \
  do {                                                                                         \
    auto kern = vcs_lanczos2_kernel<ALPHA, MINB, TH, NWC, X4>;                                 \
    static bool attr_done[16] = {false};                                                       \
    int dev = 0; cudaGetDevice (&dev);                                                         \
    if (!attr_done[dev & 15]) {                                                                \
      B200_CUDA_TRY (cudaFuncSetAttribute (kern, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
              L2Shape<TH, NWC>::SMEM));                                                        \
      attr_done[dev & 15] = true;                                                              \
    }                                                                                          \
    dim3 grid ((d.ow + L2Shape<TH, NWC>::TW - 1) / L2Shape<TH, NWC>::TW, (d.oh + TH - 1) / TH, n); \
    kern <<<grid, L2_THREADS, L2Shape<TH, NWC>::SMEM, stream>>> (d, st.dev, batch);            \
  } while (0)
  if (!st.dev.alpha_opaque) L2_LAUNCH (false, 3, 32, 2);
  else if (st.x4) L2_LAUNCH_X (true, 4, 60, 1, true);              // the default shape with taps times 4
  else switch (st.variant) {
    case 1: L2_LAUNCH (true, 4, 32, 2); break;
    case 2: L2_LAUNCH (true, 3, 60, 1); break;
    case 3: L2_LAUNCH (true, 4, 60, 1); break;
    default: L2_LAUNCH (true, 3, 32, 2); break;
  }
#undef L2_LAUNCH
#undef L2_LAUNCH_X
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
