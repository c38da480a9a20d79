// gstreamer_b200/csrc/vcs_l2tc.cuh — the exact-2:1 / 8-tap kernel with both FIR passes on the Hopper tensor cores
// (product code, sm_90a: wgmma.mma_async with s8 x u8 operands from shared memory and s32 accumulators in registers).
//
// Why: the SIMT 2:1 kernel spends most of its issue slots on the horizontal FIR's dot products and the shuffles, shifts
// and packs around them.  Both FIRs are banded u8 x s8 matrix products with exact 32-bit accumulation, so they can run
// on the tensor cores instead:
//
//   H pass   D_h[j][l] = sum_x band[j][x] * img[l][x]       A = tap band of the strip's 128 output columns (s8, K-major)
//                                                           B = the staged input lines of one channel (u8, K = pixels)
//   V pass   D_v[c][r] = sum_l hs[c][l]   * vband[r][l]     A = h-scaled samples, one row per output column (u8, K = lines)
//                                                           B = tap band of the tile's output rows (s8)
//
// Each of the two warpgroups owns 64 of the strip's 128 output columns (wgmma M = 64) in both passes, so the h-scaled
// operand a warpgroup writes after its H pass is read only by its own V pass.  Rounding is one more K step against a
// block of ones ((acc + 32) >> 6, or taps times 4 and + 128 so that the saturated result is byte 1 of a 16-bit
// saturating pack); garbage in staged samples outside the frame meets zero taps (the reference folds its edge taps
// inward, see pack of the bands below), so no clamped copies are needed.
// What stays SIMT is what is not linear: de-interleaving and the two rounding chroma up-sampling steps
// (video-chroma.c:687-699, video-orc.orc:2705-2735), saturation, and the AYUV -> ARGB mulhi matrix.
//
// Shared-memory operands use the un-swizzled canonical K-major layout (8 rows x 16 bytes = one contiguous 128-byte core
// matrix; LBO = distance of the next 16-byte K chunk, SBO = distance of the next 8 rows), which plain 16-byte stores and
// cp.async produce without any address swizzling.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

#include "common.h"
#include "vcs_device.h"
#include "vcs_plan.h"
#include "vcs_lanczos2.cuh"

namespace b200 {

constexpr int TC_THREADS = 256;                            // two warpgroups
constexpr int TC_PROD_WARPS = TC_THREADS / 32;             // every warp stages
constexpr int TC_TW = 128;                                 // output columns per tile = rows of the band (2 x wgmma M)
constexpr int TC_TH = 28;                                  // output rows per tile
constexpr int TC_N = 64;                                   // staged input lines (2 * TH + 6 = 62 used) = wgmma N of the H pass
constexpr int TC_CHUNKS = 18;                              // 16-byte chunks per staged line: 288 input bytes (2 * 128 + 6, 16-aligned start)
constexpr int TC_X_LEAD = 16;                              // the staged window starts 16 pixels left of the strip's first tap centre - 3
constexpr int TC_IMG_LBO = 8 * 128 + 16;                   // bytes between chunk columns of a staged plane (+16: bank spread)
constexpr int TC_IMG_BYTES = TC_CHUNKS * TC_IMG_LBO;       // 18 720
constexpr int TC_BAND_CHUNKS = TC_CHUNKS + 2;              // + the rounding K step
constexpr int TC_BAND_LBO = 16 * 128;                      // 128 rows
constexpr int TC_BAND_BYTES = TC_BAND_CHUNKS * TC_BAND_LBO;   // 40 960
constexpr int TC_ONES_BYTES = 2 * TC_BAND_LBO;             // [2 chunks][128 rows][16]: every byte 1
constexpr int TC_VROWS = 32;                               // wgmma N of the V pass (28 used)
constexpr int TC_VB_CHUNKS = TC_N / 16 + 2;
constexpr int TC_VB_LBO = (TC_VROWS / 8) * 128;            // 512
constexpr int TC_VB_BYTES = TC_VB_CHUNKS * TC_VB_LBO;      // 3 072
constexpr int TC_HS_LBO = 16 * 128;
constexpr int TC_HS_BYTES = (TC_N / 16) * TC_HS_LBO;       // per channel 8 192
// shared-memory map
constexpr int TC_OFF_BAND = 0;
constexpr int TC_OFF_ONES = TC_OFF_BAND + TC_BAND_BYTES;
constexpr int TC_OFF_VB = TC_OFF_ONES + TC_ONES_BYTES;
constexpr int TC_OFF_IMG = TC_OFF_VB + TC_VB_BYTES;         // 3 planes
constexpr int TC_OFF_HS = TC_OFF_IMG + 3 * TC_IMG_BYTES;    // 3 channels of the V pass's A operand
constexpr int TC_SMEM = TC_OFF_HS + 3 * TC_HS_BYTES;        // 128 864: one CTA per SM
static_assert (TC_OFF_IMG % 16 == 0 && TC_IMG_BYTES % 16 == 0 && TC_OFF_HS % 16 == 0, "operand alignment");
static_assert (TC_SMEM <= 227 * 1024, "one CTA must fit the opt-in shared memory of sm_90");

struct L2tcDev {
  const uint8_t *band;          // [strips][TC_BAND_BYTES]   tap band of each 128-column strip, canonical layout, + rounding step
  const uint8_t *vband;         // [row tiles][TC_VB_BYTES]
  const uint8_t *hx4, *vx4;     // per strip / row tile: taps are stored times 4 (rounding 128, result in byte 1)
  int strips, row_tiles;
  unsigned magic_rt;            // 2^32 / row_tiles + 1: t / row_tiles == umulhi (t, magic) for the tile counts that occur
};

// ---- PTX wrappers (sm_90a) ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t tc_smem_u32 (const void *p) { return (uint32_t) __cvta_generic_to_shared (p); }
__device__ __forceinline__ uint64_t tc_desc (uint32_t saddr, uint32_t lbo, uint32_t sbo)
{
  // wgmma matrix descriptor, no swizzle (layout 0 at bits 62-63): start >> 4 | LBO >> 4 << 16 | SBO >> 4 << 32
  return (uint64_t) ((saddr >> 4) & 0x3fffu) | ((uint64_t) ((lbo >> 4) & 0x3fffu) << 16) |
      ((uint64_t) ((sbo >> 4) & 0x3fffu) << 32);
}
__device__ __forceinline__ void tc_fence_async_smem () {
#ifndef B200_CUDA_EMU
  asm volatile ("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
__device__ __forceinline__ void tc_cp16 (uint32_t saddr, const void *g)
{
#ifndef B200_CUDA_EMU
  asm volatile ("cp.async.cg.shared.global [%0], [%1], 16;" :: "r" (saddr), "l" (g) : "memory");
#endif
}
__device__ __forceinline__ void tc_cp_wait ()
{
#ifndef B200_CUDA_EMU
  asm volatile ("cp.async.wait_all;" ::: "memory");
#endif
}
__device__ __forceinline__ void tc_wg_fence () {
#ifndef B200_CUDA_EMU
  asm volatile ("wgmma.fence.sync.aligned;" ::: "memory");
#endif
}
__device__ __forceinline__ void tc_wg_commit_wait () {
#ifndef B200_CUDA_EMU
  asm volatile ("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile ("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#endif
}
// the accumulators are written asynchronously: no use of them may be scheduled before the wait
template <int N>
__device__ __forceinline__ void tc_fence_regs (int (&d)[N])
{
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile ("" : "+r" (d[i]) :: "memory");
}

// H pass step: D (64 columns x 64 lines, s32) (+)= band (s8) x img (u8)
__device__ __forceinline__ void tc_mma_h (int (&d)[32], uint64_t adesc, uint64_t bdesc, int accumulate)
{
#ifndef B200_CUDA_EMU
  asm volatile ("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.u8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31},"
      " %32, %33, p;\n\t}\n"
      : "+r" (d[0]), "+r" (d[1]), "+r" (d[2]), "+r" (d[3]), "+r" (d[4]), "+r" (d[5]), "+r" (d[6]), "+r" (d[7]),
        "+r" (d[8]), "+r" (d[9]), "+r" (d[10]), "+r" (d[11]), "+r" (d[12]), "+r" (d[13]), "+r" (d[14]), "+r" (d[15]),
        "+r" (d[16]), "+r" (d[17]), "+r" (d[18]), "+r" (d[19]), "+r" (d[20]), "+r" (d[21]), "+r" (d[22]), "+r" (d[23]),
        "+r" (d[24]), "+r" (d[25]), "+r" (d[26]), "+r" (d[27]), "+r" (d[28]), "+r" (d[29]), "+r" (d[30]), "+r" (d[31])
      : "l" (adesc), "l" (bdesc), "r" (accumulate) : "memory");
#endif
}
// V pass step: D (64 columns x 32 rows, s32) (+)= hs (u8) x vband (s8)
__device__ __forceinline__ void tc_mma_v (int (&d)[16], uint64_t adesc, uint64_t bdesc, int accumulate)
{
#ifndef B200_CUDA_EMU
  asm volatile ("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n\t}\n"
      : "+r" (d[0]), "+r" (d[1]), "+r" (d[2]), "+r" (d[3]), "+r" (d[4]), "+r" (d[5]), "+r" (d[6]), "+r" (d[7]),
        "+r" (d[8]), "+r" (d[9]), "+r" (d[10]), "+r" (d[11]), "+r" (d[12]), "+r" (d[13]), "+r" (d[14]), "+r" (d[15])
      : "l" (adesc), "l" (bdesc), "r" (accumulate) : "memory");
#endif
}

// two consecutive FIR sums -> two rounded, saturated bytes (lowest byte = first sum); the rounding constant is already
// in the accumulator (the extra K step)
template <bool X4>
__device__ __forceinline__ unsigned short tc_pack2 (int a0, int a1)
{
  if (X4) return (unsigned short) __byte_perm (pack_sat_u16x2 (a1, a0), 0, 0x4431);
  return (unsigned short) pack_sat2 (a1 >> 6, a0 >> 6, 0u);
}

// one output pixel from the three rounded V sums: AYUV -> ARGB (mulhi matrix) -> the output byte order
template <bool X4>
__device__ __forceinline__ unsigned tc_pixel (const VcsDev & P, int y, int u, int v)
{
  unsigned yuv = X4 ? __byte_perm (pack_sat_u16x2 (u, y), pack_sat_u16x2 (0, v), 0x7531)
      : pack_sat2 (u >> 6, y >> 6, pack_sat2 (0, v >> 6, 0u));
  yuv ^= 0x00808080u;
  const int wy = prmt_s (yuv, 0x8800u), wu = prmt_s (yuv, 0x9911u), wv = prmt_s (yuv, 0xaa22u);
  const int ty = ((wy * P.p1) >> 16) + 128;
  const int r = ty + ((wv * P.p2) >> 16);
  const int b = ty + ((wu * P.p3) >> 16);
  const int gg = ty + ((wu * P.p4) >> 16) + ((wv * P.p5) >> 16);
  const unsigned argb = pack_sat2 (r, 255, pack_sat2 (b, gg, 0u));
  return __byte_perm (argb, 0, P.sel);
}

// ---- the kernel ------------------------------------------------------------------------------------------------------
// One persistent CTA per SM walks its tiles (strip, frame, row tile); per tile:
//   1. all eight warps stage the tile: tap bands and Y by cp.async, the up-sampled chroma by SIMT
//   2. each warpgroup runs the H pass of its 64 columns channel by channel and writes the rounded bytes as the V pass's
//      A operand
//   3. each warpgroup runs the V pass of its 64 columns for the three channels, then converts and stores the pixels
// wgmma fragment of D (m64nN): warp w of the warpgroup, lane = 4 g + t holds rows 16 w + g and 16 w + g + 8, columns
// 8 i + 2 t and 8 i + 2 t + 1: d[4 i + 0..3] = (g, 2t), (g, 2t + 1), (g + 8, 2t), (g + 8, 2t + 1).  In the code g is fr, t is t4.
__global__ void __launch_bounds__ (TC_THREADS, 1)
vcs_l2tc_kernel (const VcsDev P, const L2tcDev L, const VcsBatch frames, int n_frames)
{
#ifndef B200_CUDA_EMU
  extern __shared__ __align__ (128) uint8_t sm[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync (0xffffffffu, tid >> 5, 0);
  const int wg = warp >> 2, fr = lane >> 2, t4 = lane & 3;      // fr, t4: row group / pair of a wgmma fragment
  const uint32_t s_base = tc_smem_u32 (sm);
  const uint32_t s_band = s_base + TC_OFF_BAND, s_ones = s_base + TC_OFF_ONES, s_vb = s_base + TC_OFF_VB,
      s_img = s_base + TC_OFF_IMG, s_hs = s_base + TC_OFF_HS;

  for (int i = tid; i < TC_ONES_BYTES / 16; i += TC_THREADS)
    *(uint4 *) (sm + TC_OFF_ONES + 16 * i) = make_uint4 (0x01010101u, 0x01010101u, 0x01010101u, 0x01010101u);

  const int per_strip = n_frames * L.row_tiles;
  const int n_tiles = L.strips * per_strip;
  const int my_tiles = blockIdx.x < n_tiles ? (n_tiles - 1 - (int) blockIdx.x) / (int) gridDim.x + 1 : 0;
  const unsigned magic_ps = 0xffffffffu / (unsigned) per_strip + 1u;    // tiles < 2^16 * ... : exact for t < 2^32 / per_strip
  auto tile_of = [&] (int k, int & strip, int & f, int & rt) {
    const unsigned t = blockIdx.x + (unsigned) k * gridDim.x;
    strip = (int) __umulhi (t, magic_ps);
    if ((unsigned) (strip + 1) * (unsigned) per_strip <= t) strip++;          // the reciprocals round down at most one short
    const unsigned rem = t - (unsigned) strip * (unsigned) per_strip;
    f = (int) __umulhi (rem, L.magic_rt);
    if ((unsigned) (f + 1) * (unsigned) L.row_tiles <= rem) f++;
    rt = (int) (rem - (unsigned) f * (unsigned) L.row_tiles);
  };
  // descriptors differ only in their start-address field (bits 0..13, units of 16 bytes): base descriptor + offset.
  // Warpgroup wg's 64 rows of an A operand start 64 rows = 8 core matrices (1 KB) further.
  const uint64_t d_band = tc_desc (s_band + 1024u * wg, TC_BAND_LBO, 128), d_ones = tc_desc (s_ones, TC_BAND_LBO, 128);
  const uint64_t d_img = tc_desc (s_img, TC_IMG_LBO, 128), d_hs = tc_desc (s_hs + 1024u * wg, TC_HS_LBO, 128);
  const uint64_t d_vb = tc_desc (s_vb, TC_VB_LBO, 128);

  const int crows = P.ih >> 1;
  const unsigned selU = P.u_index ? 0x7531u : 0x6420u, selV = P.u_index ? 0x6420u : 0x7531u;
  const unsigned nselU = P.u_index ? 0x5321u : 0x4321u, nselV = P.u_index ? 0x4321u : 0x5321u;
  int prev_strip = -1;
  for (int k = 0; k < my_tiles; k++) {
    int strip, f, rt;
    tile_of (k, strip, f, rt);
    const int x0 = strip * TC_TW, oy0 = rt * TC_TH;
    __syncthreads ();                                              // both warpgroups are done with the previous tile's operands
    // ================================================================ 1. staging
    {
      if (strip != prev_strip) {
        const uint8_t *src = L.band + (size_t) strip * TC_BAND_BYTES;
        for (int i = tid; i < TC_BAND_BYTES / 16; i += TC_THREADS) tc_cp16 (s_band + 16 * i, src + 16 * i);
        prev_strip = strip;
      }
      const uint8_t *__restrict__ in = frames.in[f];
      const uint8_t *__restrict__ plane_y = in + P.off_y;
      const uint8_t *__restrict__ plane_c = in + P.off_c;
      const int X0 = 2 * x0 - TC_X_LEAD, R0 = 2 * oy0 - 3;
      const uint32_t img = s_img;
      uint8_t *img_u = sm + TC_OFF_IMG + TC_IMG_BYTES, *img_v = img_u + TC_IMG_BYTES;
      if (tid < TC_VB_BYTES / 16) tc_cp16 (s_vb + 16 * tid, L.vband + (size_t) rt * TC_VB_BYTES + 16 * tid);
      // Y: a warp takes lines w, w + 8, ...; lanes 0..17 one 16-byte chunk each
      {
        const int x = X0 + 16 * lane;
        const bool xin = lane < TC_CHUNKS && x >= 0 && x + 16 <= P.iw;
        const uint8_t *src = plane_y + (ptrdiff_t) (R0 + warp) * P.stride_y + x;
        const ptrdiff_t step = (ptrdiff_t) TC_PROD_WARPS * P.stride_y;
        for (int li = warp; li < 2 * TC_TH + 6; li += TC_PROD_WARPS, src += step) {
          const int y = R0 + li;
          if (xin && y >= 0 && y < P.ih) tc_cp16 (img + lane * TC_IMG_LBO + (li >> 3) * 128 + (li & 7) * 16, src);
        }
      }
      // chroma: item = (line group g, 8-pixel slot); units of 32 items, the odd unit rotates over the warps.  All raw
      // chroma of a warp's (at most 3) units is requested before the first byte-SIMD instruction needs any of it.
      {
        constexpr int SLOTS = 2 * TC_CHUNKS - 2, ITEMS = (TC_N / 4) * SLOTS, UNITS = (ITEMS + 31) / 32;
        constexpr int MAXU = (UNITS + TC_PROD_WARPS - 1) / TC_PROD_WARPS;
        const int u0 = (warp + k) % TC_PROD_WARPS;
        // tiles that touch no frame border: no row clamps, no right-edge replication, no column tests
        const bool interior = R0 >= 1 && R0 + 4 * (TC_N / 4) + 2 <= P.ih && X0 >= 0 && X0 + 16 * TC_CHUNKS + 8 <= P.iw;
        uint2 raw[MAXU][3];
        unsigned nxt[MAXU][3];
        int offs[MAXU];
        bool redge[MAXU];
#pragma unroll
        for (int j = 0; j < MAXU; j++) {
          const int item = 32 * (u0 + j * TC_PROD_WARPS) + lane;
          offs[j] = -1; redge[j] = false;
          if (u0 + j * TC_PROD_WARPS < UNITS && item < ITEMS) {
            const int g = item / SLOTS, slot = item - g * SLOTS + 1;
            const int x = X0 + 8 * slot;
            if (interior) {
              offs[j] = (slot >> 1) * TC_IMG_LBO + (g >> 1) * 128 + (g & 1) * 64 + (slot & 1) * 8;
              const uint8_t *row = plane_c + (ptrdiff_t) (oy0 - 2 + 2 * g) * P.stride_c + x;    // (R0 + 4g - 1) >> 1 == oy0 - 2 + 2g
#pragma unroll
              for (int kk = 0; kk < 3; kk++, row += P.stride_c) {
                raw[j][kk] = __ldg ((const uint2 *) row);
                nxt[j][kk] = (unsigned) __ldg ((const unsigned short *) (row + 8));
              }
            } else if (x >= 0 && x < P.iw) {
              redge[j] = x + 8 >= P.iw;
              const int m2 = (R0 + 4 * g - 1) >> 1;
              offs[j] = (slot >> 1) * TC_IMG_LBO + (g >> 1) * 128 + (g & 1) * 64 + (slot & 1) * 8;   // line 4g + r: + 16 r
#pragma unroll
              for (int kk = 0; kk < 3; kk++) {
                const int cr = min (max (m2 + kk, 0), crows - 1);
                const uint8_t *row = plane_c + (size_t) cr * P.stride_c + x;
                raw[j][kk] = __ldg ((const uint2 *) row);
                nxt[j][kk] = redge[j] ? 0u : (unsigned) __ldg ((const unsigned short *) (row + 8));
              }
            }
          }
        }
#pragma unroll
        for (int j = 0; j < MAXU; j++) {
          if (offs[j] < 0) continue;
          unsigned ulo[3], uhi[3], vlo[3], vhi[3];
#pragma unroll
          for (int kk = 0; kk < 3; kk++) {
            const uint2 c = raw[j][kk];
            const unsigned ue = __byte_perm (c.x, c.y, selU), ve = __byte_perm (c.x, c.y, selV);
            const unsigned un = redge[j] ? __byte_perm (ue, ue, 0x3321) : __byte_perm (ue, nxt[j][kk], nselU);
            const unsigned vn = redge[j] ? __byte_perm (ve, ve, 0x3321) : __byte_perm (ve, nxt[j][kk], nselV);
            const unsigned uo = avg_ceil4 (ue, un), vo = avg_ceil4 (ve, vn);
            ulo[kk] = __byte_perm (ue, uo, 0x5140); uhi[kk] = __byte_perm (ue, uo, 0x7362);
            vlo[kk] = __byte_perm (ve, vo, 0x5140); vhi[kk] = __byte_perm (ve, vo, 0x7362);
          }
          uint2 U[4], V[4];
          {
            unsigned q;
            q = avg_floor4 (ulo[0], ulo[1]); U[0].x = avg_ceil4 (ulo[0], q); U[1].x = avg_ceil4 (ulo[1], q);
            q = avg_floor4 (uhi[0], uhi[1]); U[0].y = avg_ceil4 (uhi[0], q); U[1].y = avg_ceil4 (uhi[1], q);
            q = avg_floor4 (ulo[1], ulo[2]); U[2].x = avg_ceil4 (ulo[1], q); U[3].x = avg_ceil4 (ulo[2], q);
            q = avg_floor4 (uhi[1], uhi[2]); U[2].y = avg_ceil4 (uhi[1], q); U[3].y = avg_ceil4 (uhi[2], q);
            q = avg_floor4 (vlo[0], vlo[1]); V[0].x = avg_ceil4 (vlo[0], q); V[1].x = avg_ceil4 (vlo[1], q);
            q = avg_floor4 (vhi[0], vhi[1]); V[0].y = avg_ceil4 (vhi[0], q); V[1].y = avg_ceil4 (vhi[1], q);
            q = avg_floor4 (vlo[1], vlo[2]); V[2].x = avg_ceil4 (vlo[1], q); V[3].x = avg_ceil4 (vlo[2], q);
            q = avg_floor4 (vhi[1], vhi[2]); V[2].y = avg_ceil4 (vhi[1], q); V[3].y = avg_ceil4 (vhi[2], q);
          }
#pragma unroll
          for (int r = 0; r < 4; r++) {
            *(uint2 *) (img_u + offs[j] + 16 * r) = U[r];
            *(uint2 *) (img_v + offs[j] + 16 * r) = V[r];
          }
        }
      }
      tc_cp_wait ();
      tc_fence_async_smem ();                                      // generic-proxy writes -> visible to wgmma
      __syncthreads ();
    }
    // ================================================================ 2. H pass, one channel at a time
    const bool hx4 = __ldg (L.hx4 + strip) != 0;                  // block-uniform
#pragma unroll 1
    for (int ch = 0; ch < 3; ch++) {
      int d[32];
#pragma unroll
      for (int i = 0; i < 32; i++) d[i] = 0;
      const uint64_t img = d_img + (uint64_t) ((ch * TC_IMG_BYTES) >> 4);
      tc_fence_regs (d);
      tc_wg_fence ();
#pragma unroll
      for (int s = 0; s < TC_CHUNKS / 2; s++)
        tc_mma_h (d, d_band + (uint64_t) ((2 * s * TC_BAND_LBO) >> 4), img + (uint64_t) ((2 * s * TC_IMG_LBO) >> 4), s > 0);
      tc_mma_h (d, d_band + (uint64_t) ((TC_CHUNKS * TC_BAND_LBO) >> 4), d_ones, 1);
      tc_wg_commit_wait ();
      tc_fence_regs (d);
      // rows = output columns j, columns = staged lines l: the pair (l, l + 1) is two adjacent bytes of hs row j
      uint8_t *hs = sm + TC_OFF_HS + ch * TC_HS_BYTES + (64 * wg + 16 * (warp & 3) + fr) * 16;
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int l = 8 * i + 2 * t4;
        uint8_t *p = hs + (l >> 4) * TC_HS_LBO + (l & 15);
        if (hx4) {
          *(unsigned short *) p = tc_pack2<true> (d[4 * i], d[4 * i + 1]);
          *(unsigned short *) (p + 8 * 16) = tc_pack2<true> (d[4 * i + 2], d[4 * i + 3]);
        } else {
          *(unsigned short *) p = tc_pack2<false> (d[4 * i], d[4 * i + 1]);
          *(unsigned short *) (p + 8 * 16) = tc_pack2<false> (d[4 * i + 2], d[4 * i + 3]);
        }
      }
    }
    tc_fence_async_smem ();
    __syncthreads ();
    // ================================================================ 3. V pass, the three channels together
    {
      int a[3][16];
#pragma unroll
      for (int ch = 0; ch < 3; ch++)
#pragma unroll
        for (int i = 0; i < 16; i++) a[ch][i] = 0;
      tc_fence_regs (a[0]); tc_fence_regs (a[1]); tc_fence_regs (a[2]);
      tc_wg_fence ();
#pragma unroll
      for (int ch = 0; ch < 3; ch++) {
        const uint64_t hs = d_hs + (uint64_t) ((ch * TC_HS_BYTES) >> 4);
#pragma unroll
        for (int s = 0; s < TC_N / 32; s++)
          tc_mma_v (a[ch], hs + (uint64_t) ((2 * s * TC_HS_LBO) >> 4), d_vb + (uint64_t) ((2 * s * TC_VB_LBO) >> 4), s > 0);
        tc_mma_v (a[ch], d_ones, d_vb + (uint64_t) ((2 * (TC_N / 32) * TC_VB_LBO) >> 4), 1);
      }
      tc_wg_commit_wait ();
      tc_fence_regs (a[0]); tc_fence_regs (a[1]); tc_fence_regs (a[2]);
      // rows = output columns, columns = output rows of the tile
      const bool vx4 = __ldg (L.vx4 + rt) != 0;
      uint8_t *out = frames.out[f] + P.off_out;
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const int ox = x0 + 64 * wg + 16 * (warp & 3) + fr + ((e & 2) ? 8 : 0);
        const int r = 8 * (e >> 2) + 2 * t4 + (e & 1);
        if (r < TC_TH && oy0 + r < P.oh && ox < P.ow)
          *(unsigned *) (out + (size_t) (oy0 + r) * P.stride_out + (size_t) ox * 4u) =
              vx4 ? tc_pixel<true> (P, a[0][e], a[1][e], a[2][e]) : tc_pixel<false> (P, a[0][e], a[1][e], a[2][e]);
      }
    }
  }
#endif
}

// ------------------------------------------------------------------------------------------------------- host side
struct L2tcTables {
  std::vector<uint8_t> band, vband, hx4, vx4;
  int strips = 0, row_tiles = 0;
  bool ok = false;
};

// canonical K-major byte position of element (row, k) in an operand whose 16-byte K chunks are `lbo` apart
inline size_t tc_pos (int row, int k, int lbo) { return (size_t) (k >> 4) * lbo + (size_t) row * 16 + (k & 15); }

inline L2tcTables build_l2tc_tables (const VcsPlan & p, const Lanczos2Tables & l2)
{
  L2tcTables t;
  if (!l2.ok || !l2.alpha_opaque || p.planar) return t;           // same eligibility as the SIMT 2:1 kernel, opaque alpha, semi-planar only
  if ((p.in.width & 15) || (p.in.stride[0] & 15) || (p.in.stride[1] & 15) || (p.in.offset[0] & 15) || (p.in.offset[1] & 15)) return t;
  const int ow = p.out.width, oh = p.out.height, iw = p.in.width, ih = p.in.height;
  t.strips = (ow + TC_TW - 1) / TC_TW; t.row_tiles = (oh + TC_TH - 1) / TC_TH;
  t.band.assign ((size_t) t.strips * TC_BAND_BYTES, 0); t.hx4.assign (t.strips, 1);
  t.vband.assign ((size_t) t.row_tiles * TC_VB_BYTES, 0); t.vx4.assign (t.row_tiles, 1);
  for (int s = 0; s < t.strips; s++) {
    const int x0 = s * TC_TW, X0 = 2 * x0 - TC_X_LEAD;
    for (int j = 0; j < TC_TW && x0 + j < ow; j++)
      for (int k = 0; k < 8; k++) { const int v = 4 * p.h.coef[(size_t) (x0 + j) * 8 + k]; if (v < -128 || v > 127) t.hx4[s] = 0; }
    const int scale = t.hx4[s] ? 4 : 1;
    uint8_t *b = t.band.data () + (size_t) s * TC_BAND_BYTES;
    for (int j = 0; j < TC_TW; j++) {
      b[tc_pos (j, 16 * TC_CHUNKS, TC_BAND_LBO)] = (uint8_t) (t.hx4[s] ? 127 : 32);     // rounding step against the ones block ...
      if (t.hx4[s]) b[tc_pos (j, 16 * TC_CHUNKS + 1, TC_BAND_LBO)] = 1;                // ... 127 + 1 = 128 (s8 holds no 128)
      if (x0 + j >= ow) continue;
      for (int k = 0; k < 8; k++) {
        const int tap = p.h.coef[(size_t) (x0 + j) * 8 + k];
        if (!tap) continue;
        const int xr = (int) p.h.offset[x0 + j] + k - X0;
        if (xr < 0 || xr >= 16 * TC_CHUNKS || (int) p.h.offset[x0 + j] + k >= iw) return t;
        b[tc_pos (j, xr, TC_BAND_LBO)] = (uint8_t) (int8_t) (scale * tap);
      }
    }
  }
  for (int rt = 0; rt < t.row_tiles; rt++) {
    const int oy0 = rt * TC_TH, R0 = 2 * oy0 - 3;
    for (int r = 0; r < TC_TH && oy0 + r < oh; r++)
      for (int k = 0; k < 8; k++) { const int v = 4 * p.v.coef[(size_t) (oy0 + r) * 8 + k]; if (v < -128 || v > 127) t.vx4[rt] = 0; }
    const int scale = t.vx4[rt] ? 4 : 1;
    uint8_t *b = t.vband.data () + (size_t) rt * TC_VB_BYTES;
    for (int r = 0; r < TC_VROWS; r++) {
      b[tc_pos (r, TC_N, TC_VB_LBO)] = (uint8_t) (t.vx4[rt] ? 127 : 32);
      if (t.vx4[rt]) b[tc_pos (r, TC_N + 1, TC_VB_LBO)] = 1;
      if (r >= TC_TH || oy0 + r >= oh) continue;
      for (int k = 0; k < 8; k++) {
        const int tap = p.v.coef[(size_t) (oy0 + r) * 8 + k];
        if (!tap) continue;
        const int li = (int) p.v.offset[oy0 + r] + k - R0;
        if (li < 0 || li >= 2 * TC_TH + 6 || (int) p.v.offset[oy0 + r] + k >= ih) return t;
        b[tc_pos (r, li, TC_VB_LBO)] = (uint8_t) (int8_t) (scale * tap);
      }
    }
  }
  t.ok = true;
  return t;
}

struct L2tcState {
  uint8_t *d_band = nullptr, *d_vband = nullptr, *d_hx4 = nullptr, *d_vx4 = nullptr;
  L2tcDev dev;
  bool ready = false;
};

inline int prepare_l2tc (const L2tcTables & t, L2tcState * st)
{
  int rc;
  if (!t.ok) return B200_OK;
  if ((rc = upload (&st->d_band, t.band.data (), t.band.size ())) != B200_OK) return rc;
  if ((rc = upload (&st->d_vband, t.vband.data (), t.vband.size ())) != B200_OK) return rc;
  if ((rc = upload (&st->d_hx4, t.hx4.data (), t.hx4.size ())) != B200_OK) return rc;
  if ((rc = upload (&st->d_vx4, t.vx4.data (), t.vx4.size ())) != B200_OK) return rc;
  st->dev.band = st->d_band; st->dev.vband = st->d_vband; st->dev.hx4 = st->d_hx4; st->dev.vx4 = st->d_vx4;
  st->dev.strips = t.strips; st->dev.row_tiles = t.row_tiles;
  st->dev.magic_rt = 0xffffffffu / (unsigned) t.row_tiles + 1u;
  st->ready = true;
  return B200_OK;
}

inline int launch_l2tc (const VcsDev & d, const L2tcState & st, const VcsBatch & batch, int n, cudaStream_t stream)
{
  int rc;
  int dev = 0;
  B200_CUDA_TRY (cudaGetDevice (&dev));
  const int tiles = st.dev.strips * st.dev.row_tiles * n;
  const int grid = min (tiles, sm_count (dev));
  static bool attr_done[16] = {false};
  if (!attr_done[dev & 15]) {
    if ((rc = allow_max_dyn_smem (vcs_l2tc_kernel)) != B200_OK) return rc;
    attr_done[dev & 15] = true;
  }
  vcs_l2tc_kernel <<<grid, TC_THREADS, TC_SMEM, stream>>> (d, st.dev, batch, n);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
