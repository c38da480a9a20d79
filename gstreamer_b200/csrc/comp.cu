// gstreamer_b200/csrc/comp.cu — b200_comp_* : single-pass compositor (product code, sm_90a).
//
// Replaces the per-pad read-modify-write passes of the reference
//   blend_pads()/_draw_background()      gst-plugins-base/gst/compositor/compositor.c:1619-1697
//   BLEND_A32 clip + _blend_loop/_overlay_loop   gst/compositor/blend.c:42-159
//   compositor_orc_{blend,source,overlay,overlay_*_addition}_{argb,bgra}   compositororc.orc:163-560
// with ONE kernel: every output pixel starts from the background value, walks the pads that
// cover it in z-order entirely in registers, and is written once.  Bytes are identical to the
// sequential reference because each pad's operator only reads the destination pixel it writes.
//
// HBM traffic per frame = every covered source pixel once + the destination once
// (the reference moves bg write + per pad src read + dst read + dst write).
#include "common.h"
#include "video_format.h"
#include "vcs_device.h"

#include <string.h>
#include <algorithm>
#include <new>

namespace b200 {

enum CompMode : int { CM_COPY = 0, CM_SOURCE = 1, CM_BLEND = 2, CM_OVERLAY = 3, CM_OVERLAY_ADD = 4 };

struct CompPadDev {
  const uint8_t *data;           // already offset so that data + y*stride + x*4 addresses DEST pixel (x,y)
  long long stride;
  int x0, y0, x1, y1;            // clipped destination rectangle
  int s_alpha, mode;
};

constexpr int COMP_CHUNK = 32;

struct CompParams {
  uint8_t *dst;
  int width, height, stride;
  int background;                // b200_comp_background, or -1: continue from the current dst contents
  int alpha_shift;               // bit position of the alpha byte in a little-endian pixel word (0 or 24)
  int n_pads;
  int need_recip;                // some pad uses the overlay family (needs the reciprocal table)
  CompPadDev pads[COMP_CHUNK];
};

// floor(x/255) on two 16-bit lanes, x <= 65025 per lane (== div255w: (x*0x8081)>>23, compositororc.orc)
__device__ __forceinline__ unsigned div255_x2 (unsigned t)
{
  return ((t + 0x00010001u + ((t >> 8) & 0x00ff00ffu)) >> 8) & 0x00ff00ffu;
}
__device__ __forceinline__ unsigned div255_1 (unsigned x) { return (x * 0x8081u) >> 23; }

// compositor_orc_blend_*: d = div255 (s*a + d*(255-a)) on all four bytes, then alpha := 0xff.
// Two 16-bit lanes per register; floor(x/255) == (x + 1 + (x >> 8)) >> 8 for x <= 65025, and the
// final ">> 8" of both registers plus their interleave is a single PRMT.
__device__ __forceinline__ unsigned px_blend (unsigned d, unsigned s, unsigned a, unsigned alpha_mask)
{
  const unsigned ia = a ^ 0xffu;
  const unsigned se = s & 0x00ff00ffu, so = __byte_perm (s, 0, 0x4341);      // bytes 0,2 / bytes 1,3
  const unsigned de = d & 0x00ff00ffu, dd = __byte_perm (d, 0, 0x4341);
  const unsigned lo = se * a + de * ia, hi = so * a + dd * ia;               // lanes <= 65025
  const unsigned lo2 = lo + 0x00010001u + __byte_perm (lo, 0, 0x4341);
  const unsigned hi2 = hi + 0x00010001u + __byte_perm (hi, 0, 0x4341);
  return __byte_perm (lo2, hi2, 0x7351) | alpha_mask;
}

// d = { c[15:0], sat_u8(a), sat_u8(b) }  (b in the lowest byte): I2IP
__device__ __forceinline__ unsigned sat_pack2 (unsigned a, unsigned b, unsigned c)
{
#ifdef B200_CUDA_EMU               // host build of the kernel sources for tests/cudaemu: same function, plain C
  return (c << 16) | ((unsigned) min (max ((int) a, 0), 255) << 8) | (unsigned) min (max ((int) b, 0), 255);
#else
  unsigned d;
  asm ("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r" (d) : "r" (a), "r" (b), "r" (c));
  return d;
#endif
}

// compositor_orc_overlay_* (+ _addition): colour = (s*as + d*ad) / (as+ad) with divluw semantics
// (quotient clamped to 255, x/0 = 255); the alpha byte becomes as+ad (or dalpha+as, wrapping).
__device__ __forceinline__ unsigned px_overlay (unsigned d, unsigned s, unsigned as, int shift, bool addition,
    const unsigned *recip)
{
  const unsigned asel = 0x4440u | ((unsigned) shift >> 3);
  const unsigned dalpha = __byte_perm (d, 0, asel);
  const unsigned ad = div255_1 (dalpha * (as ^ 0xffu));
  const unsigned asum = as + ad;                                   // <= 255
  const unsigned se = s & 0x00ff00ffu, so = __byte_perm (s, 0, 0x4341);
  const unsigned de = d & 0x00ff00ffu, dd = __byte_perm (d, 0, 0x4341);
  const unsigned lo = se * as + de * ad, hi = so * as + dd * ad;   // lanes <= 65025: bytes (0,2) and (1,3)
  const unsigned r = recip[asum];                                  // ceil (2^24 / asum): exact floor for v < 2^16
  // umulhi (v << 8, r) == v / asum; the four "v << 8" come straight out of the lanes by PRMT
  const unsigned q0 = __umulhi (__byte_perm (lo, 0, 0x4104), r), q2 = __umulhi (__byte_perm (lo, 0, 0x4324), r);
  const unsigned q1 = __umulhi (__byte_perm (hi, 0, 0x4104), r), q3 = __umulhi (__byte_perm (hi, 0, 0x4324), r);
  unsigned out = sat_pack2 (q1, q0, sat_pack2 (q3, q2, 0u));
  if (asum == 0) out = 0xffffffffu;                                // divluw: divide by zero -> 255
  const unsigned na = addition ? dalpha + as : asum;
  return __byte_perm (out, na, shift ? 0x4210u : 0x3214u);         // alpha byte := low byte of na
}

// one pad applied to one pixel value held in a register
__device__ __forceinline__ unsigned apply_pad (unsigned d, unsigned s, int mode, unsigned s_alpha, int shift,
    unsigned alpha_mask, const unsigned *recip)
{
  if (mode == CM_COPY) return s;
  unsigned a = (s >> shift) & 0xffu;
  if (s_alpha != 255u) a = div255_1 (a * s_alpha);                 // div255 (A * 255) == A
  switch (mode) {
    case CM_SOURCE: return (s & ~alpha_mask) | (a << shift);
    case CM_BLEND: return px_blend (d, s, a, alpha_mask);
    case CM_OVERLAY: return px_overlay (d, s, a, shift, false, recip);
    default: return px_overlay (d, s, a, shift, true, recip);
  }
}

// the same for a thread's four pixels: the (warp-uniform) operator and pad-alpha tests are taken
// once, the common blend operator gets a straight-line body
__device__ __forceinline__ void apply_pad4 (unsigned (&d)[4], const unsigned (&s)[4], int mode, unsigned s_alpha,
    int shift, unsigned alpha_mask, const unsigned *recip)
{
  if (mode == CM_BLEND) {
    const unsigned asel = 0x4440u | ((unsigned) shift >> 3);        // PRMT selector: alpha byte, zero-extended
    if (s_alpha == 255u) {
#pragma unroll
      for (int i = 0; i < 4; i++) d[i] = px_blend (d[i], s[i], __byte_perm (s[i], 0, asel), alpha_mask);
    } else {
#pragma unroll
      for (int i = 0; i < 4; i++) d[i] = px_blend (d[i], s[i], div255_1 (__byte_perm (s[i], 0, asel) * s_alpha), alpha_mask);
    }
  } else if (mode == CM_COPY) {
#pragma unroll
    for (int i = 0; i < 4; i++) d[i] = s[i];
  } else {
#pragma unroll
    for (int i = 0; i < 4; i++) d[i] = apply_pad (d[i], s[i], mode, s_alpha, shift, alpha_mask, recip);
  }
}

__device__ __forceinline__ unsigned background_px (int bg, int x, int y, unsigned alpha_mask)
{
  switch (bg) {
    case B200_COMP_BG_CHECKER:                                     // fill_checker_*_c, blend.c:178-215
      return (((((y >> 3) ^ (x >> 3)) & 1) ? 160u : 80u) * 0x01010101u) | alpha_mask;
    case B200_COMP_BG_BLACK: return alpha_mask;                    // fill_color_*, blend.c:222-237
    case B200_COMP_BG_WHITE: return 0xffffffffu;
    default: return 0u;                                            // transparent: memset 0, compositor.c:1641-1672
  }
}

// tile: 128 x 8 pixels, 4 horizontally adjacent pixels per thread (16 B: one STG.128 per thread,
// LDG.128 per covering pad when the pad's x offset keeps 16 B alignment)
constexpr int CT_W = 128, CT_RPT = 1, CT_H = 8 * CT_RPT;   // 8 warps, each thread 4 pixels of CT_RPT rows (1 measured best: finer pad culling)

// what a thread needs of a pad that touches its tile, staged once per CTA (warp-uniform LDS.128 x 2
// instead of indexed constant-bank loads per thread)
struct __align__ (16) CompTilePad {
  const uint8_t *data;           // as CompPadDev::data
  long long stride;
  int x0, x1;                    // clipped destination rectangle
  int y0, y1;
  int s_alpha, mode;
  int full;                      // the whole tile lies inside the rectangle: no per-thread clipping
  int pad_;
};

__global__ void __launch_bounds__ (256)
comp_kernel (const CompParams P)
{
  __shared__ int s_count;
  __shared__ unsigned s_recip[256];
  __shared__ CompTilePad s_pads[COMP_CHUNK];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int x0 = blockIdx.x * CT_W + tx * 4, ybase = blockIdx.y * CT_H + ty;
  if (P.need_recip)                                                // only the overlay family divides
    s_recip[threadIdx.x] = threadIdx.x ? (0x1000000u + threadIdx.x - 1) / threadIdx.x : 0u;
  if (threadIdx.x < 32) {
    // which pads touch this tile?  (the reference culls whole pads, compositor.c:519-601;
    // here the cull is per tile and costs one ballot); the hits are compacted in z-order
    bool hit = false;
    const int bx = blockIdx.x * CT_W, by = blockIdx.y * CT_H;
    if ((int) threadIdx.x < P.n_pads) {
      const CompPadDev & p = P.pads[threadIdx.x];
      hit = p.x0 < bx + CT_W && p.x1 > bx && p.y0 < by + CT_H && p.y1 > by;
    }
    const unsigned m = __ballot_sync (0xffffffffu, hit);
    if (hit) {
      const CompPadDev & p = P.pads[threadIdx.x];
      CompTilePad t;
      t.data = p.data; t.stride = p.stride; t.x0 = p.x0; t.x1 = p.x1; t.y0 = p.y0; t.y1 = p.y1;
      t.s_alpha = p.s_alpha; t.mode = p.mode;
      t.full = p.x0 <= bx && p.x1 >= min (bx + CT_W, P.width) && p.y0 <= by && p.y1 >= min (by + CT_H, P.height);
      t.pad_ = 0;
      s_pads[__popc (m & ((1u << threadIdx.x) - 1u))] = t;
    }
    if (threadIdx.x == 0) s_count = __popc (m);
  }
  __syncthreads ();
  if (x0 >= P.width) return;
  const int count = s_count;
  for (int rr = 0; rr < CT_RPT; rr++) {
  const int y = ybase + 8 * rr;
  if (y >= P.height) break;
  const int n = min (4, P.width - x0);
  unsigned *dp = (unsigned *) (P.dst + (size_t) y * P.stride) + x0;
  const bool vec = n == 4 && ((((size_t) dp) & 15) == 0);
  const unsigned alpha_mask = 0xffu << P.alpha_shift;
  const int shift = P.alpha_shift;
  unsigned d[4];
  if (P.background >= 0) {
#pragma unroll
    for (int i = 0; i < 4; i++) d[i] = background_px (P.background, x0 + i, y, alpha_mask);
  } else if (vec) {                                                // continuation chunk: start from dst
    const uint4 v = *(const uint4 *) dp;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  } else {
#pragma unroll
    for (int i = 0; i < 4; i++) d[i] = i < n ? dp[i] : 0u;
  }
  // (fetching the next covering pad's pixels while the current one is blended was tried and dropped:
  //  40 registers instead of 32 cost more occupancy than the overlap returned)
  for (int k = 0; k < count; k++) {
    const CompTilePad & p = s_pads[k];
    const int full = p.full;
    if (!full && (y < p.y0 || y >= p.y1 || x0 >= p.x1 || x0 + n <= p.x0)) continue;
    const unsigned *sp = (const unsigned *) (p.data + (long long) y * p.stride) + x0;
    const int mode = p.mode;
    const unsigned s_alpha = (unsigned) p.s_alpha;
    if (n == 4 && (full || (x0 >= p.x0 && x0 + 4 <= p.x1))) {     // whole group inside the pad
      unsigned s[4];
      if ((((size_t) sp) & 15) == 0) {
        const uint4 v = __ldg ((const uint4 *) sp);
        s[0] = v.x; s[1] = v.y; s[2] = v.z; s[3] = v.w;
      } else {
#pragma unroll
        for (int i = 0; i < 4; i++) s[i] = __ldg (sp + i);
      }
      apply_pad4 (d, s, mode, s_alpha, shift, alpha_mask, s_recip);
    } else {
#pragma unroll
      for (int i = 0; i < 4; i++)
        if (i < n && x0 + i >= p.x0 && x0 + i < p.x1)
          d[i] = apply_pad (d[i], __ldg (sp + i), mode, s_alpha, shift, alpha_mask, s_recip);
    }
  }
  if (vec) {
    *(uint4 *) dp = make_uint4 (d[0], d[1], d[2], d[3]);
  } else {
#pragma unroll
    for (int i = 0; i < 4; i++) if (i < n) dp[i] = d[i];
  }
  }
}

// ------------------------------------------------------------------------------------------
// 4:2:0 output (I420 / YV12 / NV12 / NV21): blend.c PLANAR_YUV_BLEND (:246-401) and NV_YUV_BLEND
// (:1386-1500).  Per plane the reference runs compositor_orc_blend_u8 (compositororc.orc:20-36) —
// d = (d*256 + (s-d)*alpha) >> 8 on bytes, or a row copy for alpha 1.0 / SOURCE — over a byte
// rectangle; the interleaved UV plane is blended as 2*width bytes.  The host reproduces the
// reference's rectangle arithmetic (ROUND_UP_2 of the position, ceil-halved chroma extents); the
// kernel is the same single pass as comp_kernel: background, every pad in z-order in registers,
// one store, 4 bytes per thread, one launch for all planes (blockIdx.z).
constexpr int CY_MAX_PADS = 24;

struct CompYuvRect {
  const uint8_t *src;            // offset so that src + y*stride + x is the source byte of PLANE byte (x,y)
  int stride;
  int x0, x1, y0, y1;            // plane-byte rectangle
  int alpha;                     // 0 .. 2^nbits - 1 blend, CY_COPY = copy
};
constexpr int CY_COPY = 0x10000;

struct CompYuvParams {
  uint8_t *dst[3];
  int stride[3], wbytes[3], rows[3];
  int bg_mode[3];                // 0 checker (luma), 1 constant, -1 keep destination (continuation chunk)
  int bg_value[3];
  int n_planes, n_pads;
  int es, nbits;                 // bytes per sample (1, or 2: little-endian 10 / 12 / 16-bit planes), significant bits
  CompYuvRect pads[CY_MAX_PADS][3];
};

__global__ void __launch_bounds__ (256)
comp_yuv_kernel (const CompYuvParams P)
{
  const int z = blockIdx.z;
  const int x = (blockIdx.x * 32 + (threadIdx.x & 31)) * 4, y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= P.wbytes[z] || y >= P.rows[z]) return;
  uint8_t *dp = P.dst[z] + (size_t) y * P.stride[z] + x;
  const int n = min (4, P.wbytes[z] - x);
  const bool vec = n == 4 && (((size_t) dp) & 3) == 0;
  const bool wide = P.es == 2;                                     // two 16-bit samples per word
  unsigned d;
  if (P.bg_mode[z] == 0) {                                         // fill_checker_*: 8x8 squares of 80 / 160 (<< nbits - 8)
    const int px = wide ? x >> 1 : x;                              // x % 4 == 0: the word's samples share a square
    const unsigned v = (((y >> 3) ^ (px >> 3)) & 1 ? 160u : 80u) << (P.nbits - 8);
    d = wide ? v * 0x00010001u : v * 0x01010101u;
  } else if (P.bg_mode[z] == 1) {
    d = (unsigned) P.bg_value[z] * (wide ? 0x00010001u : 0x01010101u);
  } else if (vec) {
    d = *(const unsigned *) dp;
  } else {
    d = 0;
    for (int i = 0; i < n; i++) d |= (unsigned) dp[i] << (8 * i);
  }
  for (int k = 0; k < P.n_pads; k++) {
    const CompYuvRect & r = P.pads[k][z];
    if (y < r.y0 || y >= r.y1 || x >= r.x1 || x + 4 <= r.x0) continue;
    const uint8_t *sp = r.src + (size_t) y * r.stride + x;
    unsigned s = 0, m = 0;
#pragma unroll
    for (int i = 0; i < 4; i++)
      if (x + i >= r.x0 && x + i < r.x1) {
        s |= (unsigned) __ldg (sp + i) << (8 * i);
        m |= 0xffu << (8 * i);
      }
    unsigned v = s;
    if (r.alpha != CY_COPY && wide) {
      // compositor_orc_blend_u10 / _u12 / _u16 (compositororc.orc:38-100): ((d << n) + (s - d) * a) >> n in wrapping 32-bit
      // arithmetic with a logical shift, then signed-to-unsigned-word saturation
      const unsigned a = (unsigned) r.alpha;
      const unsigned d0 = d & 0xffffu, d1 = d >> 16, s0 = s & 0xffffu, s1 = s >> 16;
      const int r0 = (int) (((d0 << P.nbits) + (s0 - d0) * a) >> P.nbits), r1 = (int) (((d1 << P.nbits) + (s1 - d1) * a) >> P.nbits);
      v = (unsigned) min (max (r0, 0), 65535) | ((unsigned) min (max (r1, 0), 65535) << 16);
    } else if (r.alpha != CY_COPY) {                               // (d*(256-a) + s*a) >> 8 on two 16-bit lanes
      const unsigned a = (unsigned) r.alpha, ia = 256u - a;
      const unsigned lo = (d & 0x00ff00ffu) * ia + (s & 0x00ff00ffu) * a;
      const unsigned hi = __byte_perm (d, 0, 0x4341) * ia + __byte_perm (s, 0, 0x4341) * a;
      v = __byte_perm (lo, hi, 0x7351);
    }
    d = (v & m) | (d & ~m);
  }
  if (vec) *(unsigned *) dp = d;
  else
    for (int i = 0; i < n; i++) dp[i] = (uint8_t) (d >> (8 * i));
}

}  // namespace b200

using namespace b200;

struct b200_comp {
  int format, width, height, device;
  int alpha_shift;
  // system-memory peers (b200_comp_blend_host*): each slot holds the staged pads (in) and the destination (out) of one frame
  static const int kSlots = 3;
  HostRing<kSlots> ring;
  uint8_t *d_conv = nullptr;     // b200_comp_blend_convert: the two-pass pads' converted frames
  size_t conv_cap = 0;
};

// The 4:2:0 compositor's launches (b200_comp_blend_yuv, b200_comp_blend_convert): pads are collected in z-order and flushed
// in chunks of CY_MAX_PADS; the first launch draws the background, later ones continue from the destination.
struct YuvBlend {
  b200_comp *h = nullptr;
  CompYuvParams P;
  dim3 grid;
  cudaStream_t stream = nullptr;
  int launched = 0;
  int W = 0, H = 0, ws = 0, hs = 0, xr = 1, yr = 1, es = 1, nbits = 8, n_planes = 0;
  bool semi = false;

  static int sub (int v, int sh) { return -((-v) >> sh); }        // GST_VIDEO_FORMAT_INFO_SCALE_WIDTH / _HEIGHT (round up)

  int init (b200_comp * hh, void *dst, const b200_video_info * di, int background, cudaStream_t s)
  {
    h = hh; stream = s;
    // the format's PLANAR_YUV_BLEND / NV_YUV_BLEND instantiation (blend.c:591-646, :1386): chroma sub-sampling shifts,
    // bytes per sample and depth from the format table; the position rounds up to the chroma grid (x_round / y_round)
    const b200::VideoFormatDesc & d = *b200::video_format (h->format);
    semi = d.family == b200::FAMILY_NV;
    ws = d.wsub; hs = d.hsub; xr = 1 << ws; yr = 1 << hs; es = d.bytes; nbits = d.depth;
    W = h->width; H = h->height; n_planes = d.n_planes;
    memset (&P, 0, sizeof (P));
    P.n_planes = n_planes; P.es = es; P.nbits = nbits;
    for (int p = 0; p < n_planes; p++) {
      P.dst[p] = (uint8_t *) dst + di->offset[p];
      P.stride[p] = di->stride[p];
      P.wbytes[p] = (p == 0 ? W : (semi ? 2 * sub (W, ws) : sub (W, ws))) * es;
      P.rows[p] = p == 0 ? H : sub (H, hs);
      if (P.stride[p] < P.wbytes[p]) return B200_ERR_INVALID_ARG;
      if (es == 2 && ((P.stride[p] & 1) || (di->offset[p] & 1))) return B200_ERR_INVALID_ARG;
      // _draw_background (compositor.c:1619-1675): checker = luma squares + mid-grey chroma; black / white from the range
      // offsets at the format's depth (compositor.c:1131-1149, gst_video_color_range_offsets video-color.c:204-252: 16-235 ->
      // 16 << (n - 8) .. 235 << (n - 8); 0-255 -> 0 .. 2^n - 1; chroma 1 << (n - 1)); transparent = zeroed planes
      const bool full_range = di->color_range == B200_COLOR_RANGE_0_255;
      const int mid = 1 << (nbits - 1);
      if (background == B200_COMP_BG_CHECKER) { P.bg_mode[p] = p == 0 ? 0 : 1; P.bg_value[p] = mid; }
      else if (background == B200_COMP_BG_TRANSPARENT) { P.bg_mode[p] = 1; P.bg_value[p] = 0; }
      else {
        P.bg_mode[p] = 1;
        P.bg_value[p] = p ? mid : (background == B200_COMP_BG_BLACK ? (full_range ? 0 : 16 << (nbits - 8))
                                                                    : (full_range ? (1 << nbits) - 1 : 235 << (nbits - 8)));
      }
    }
    unsigned gx = 0, gy = 0;
    for (int p = 0; p < n_planes; p++) {
      gx = std::max (gx, (unsigned) ((P.wbytes[p] + 127) / 128));
      gy = std::max (gy, (unsigned) ((P.rows[p] + 7) / 8));
    }
    grid = dim3 (gx, gy, n_planes);
    return B200_OK;
  }

  int flush ()
  {
    comp_yuv_kernel <<<grid, 256, 0, stream>>> (P);
    B200_CUDA_TRY (cudaGetLastError ());
    launched++;
    P.n_pads = 0;
    for (int p = 0; p < n_planes; p++) P.bg_mode[p] = -1;           // later chunks continue from the destination
    return B200_OK;
  }

  // the blend's alpha of a pad: 0 = skipped, CY_COPY = copied (alpha 1.0, or SOURCE: _blend_* copies in source mode)
  int pad_alpha (double alpha, int op) const
  {
    if (op == B200_COMP_OP_SOURCE) alpha = 1.0;
    if (alpha == 0.0) return 0;
    if (alpha == 1.0) return CY_COPY;
    const int range = (1 << nbits) - 1;
    const int a = (int) (alpha * range);
    return a < 0 ? 0 : (a > range ? range : a);
  }

  // blend_<format> (blend.c:284-340 / :1418-1470): the position rounded UP to the format's grid; false when the pad lies
  // outside the frame.  x0 .. y1: the luma rectangle it covers.
  bool place (int xpos_in, int ypos_in, int w, int hgt, int *xpos, int *ypos, int *x0, int *y0, int *x1, int *y1) const
  {
    *xpos = (xpos_in + xr - 1) & ~(xr - 1); *ypos = (ypos_in + yr - 1) & ~(yr - 1);
    *x0 = std::max (*xpos, 0); *y0 = std::max (*ypos, 0);
    *x1 = std::min (*xpos + w, W); *y1 = std::min (*ypos + hgt, H);
    return *x1 > *x0 && *y1 > *y0;
  }

  int add (const void *data, const b200_video_info & info, int xpos_in, int ypos_in, double alpha, int op)
  {
    const int b_alpha = pad_alpha (alpha, op);
    if (b_alpha == 0) return B200_OK;
    int xpos, ypos, x0, y0, x1, y1;
    if (!place (xpos_in, ypos_in, info.width, info.height, &xpos, &ypos, &x0, &y0, &x1, &y1)) return B200_OK;
    const int xoffset = x0 - xpos, yoffset = y0 - ypos, bw = x1 - x0, bh = y1 - y0;
    xpos = x0; ypos = y0;
    if (P.n_pads == CY_MAX_PADS) { int st = flush (); if (st != B200_OK) return st; }
    // chroma: widths and x positions by SCALE_WIDTH (round up), rows by a plain shift (blend.c:371-376)
    const int cw = sub (bw, ws), ch = sub (bh, hs);
    const int cxpos = xpos ? sub (xpos, ws) : 0, cypos = ypos >> hs, cxoff = xoffset ? sub (xoffset, ws) : 0, cyoff = yoffset >> hs;
    for (int p = 0; p < n_planes; p++) {
      CompYuvRect & r = P.pads[P.n_pads][p];
      const int mul = ((p && semi) ? 2 : 1) * es;                   // plane bytes per (chroma) sample position
      const int px = p ? mul * cxpos : es * xpos, py = p ? cypos : ypos, sx = p ? mul * cxoff : es * xoffset, sy = p ? cyoff : yoffset;
      const int w = p ? mul * cw : es * bw, hgt = p ? ch : bh;
      r.stride = info.stride[p];
      if (es == 2 && ((r.stride & 1) || (info.offset[p] & 1) || (((uintptr_t) data) & 1))) return B200_ERR_INVALID_ARG;
      r.x0 = px; r.x1 = px + w; r.y0 = py; r.y1 = py + hgt; r.alpha = b_alpha;
      r.src = (const uint8_t *) data + info.offset[p] + (long long) (sy - py) * r.stride + (sx - px);
    }
    P.n_pads++;
    return B200_OK;
  }

  // the pads collected so far; the background alone when nothing was launched yet
  int finish () { return P.n_pads > 0 || launched == 0 ? flush () : B200_OK; }
};


// How b200_comp_blend_convert treats a pad
enum PadRoute { PR_SKIP, PR_BLEND, PR_FUSED, PR_TWO_PASS };

// The one place that decides it, from the pad's converter (none, or whether its plan scales planes into the output's
// 8-bit 4:2:0 format: vcs_comp_fusable), the output family, the alpha the blend would use (0: dropped, before any
// conversion, compositor.c:547-550) and whether the pad's clipped rectangle is empty
PadRoute pad_route (const b200_vcs * conv, bool yuv420_out, int blend_alpha, bool visible)
{
  if (blend_alpha == 0 || !visible) return PR_SKIP;
  if (!conv) return PR_BLEND;                                      // comp_kernel / comp_yuv_kernel, as b200_comp_blend[_yuv]
  if (yuv420_out && b200::vcs_comp_fusable (conv)) return PR_FUSED;   // the plane scalers store into the destination
  return PR_TWO_PASS;                                              // b200_vcs_convert_batch into d_conv, then the blend kernel
}

// The staging both host entry points share: pad i's `bytes[i]` get a 256-byte aligned place in the slot's pad buffer
// and travel up where `up[i]`; `blend` runs on the run stream over the pads' device copies; the destination comes back
// (and with `dst_up` first travels up).  The entry points have checked the arguments and set the ring up.
template <typename Pad, typename Blend>
static int comp_host_submit (b200_comp * h, void *dst_host, size_t dst_bytes, bool dst_up, const Pad * pads, int n_pads,
    const size_t * bytes, const bool * up, Blend blend)
{
  size_t need = 0, off[B200_COMP_MAX_PADS];
  for (int i = 0; i < n_pads; i++) {
    off[i] = need;
    need += (bytes[i] + 255) & ~(size_t) 255;
  }
  auto & r = h->ring;
  B200_CUDA_TRY (r.take (need, need, dst_bytes, dst_bytes));
  Pad dev_pads[B200_COMP_MAX_PADS];
  for (int i = 0; i < n_pads; i++) {
    dev_pads[i] = pads[i];
    dev_pads[i].data = r.in () + off[i];
    if (up[i]) B200_CUDA_TRY (r.upload (r.in () + off[i], pads[i].data, bytes[i]));
  }
  B200_CUDA_TRY (r.inputs_ready ());
  if (dst_up) B200_CUDA_TRY (cudaMemcpyAsync (r.out (), dst_host, dst_bytes, cudaMemcpyHostToDevice, r.run_stream ()));
  const int st = blend (r.out (), dev_pads, r.run_stream ());
  if (st != B200_OK) return st;
  B200_CUDA_TRY (r.run_done ());
  B200_CUDA_TRY (r.download (dst_host, r.out (), dst_bytes));
  B200_CUDA_TRY (r.finish ());
  return B200_OK;
}

extern "C" {

int b200_comp_create (int out_format, int width, int height, int device, b200_comp ** handle)
{
  if (!handle) return B200_ERR_INVALID_ARG;
  *handle = nullptr;
  if (width < 1 || height < 1 || width > 32767 || height > 32767) return B200_ERR_INVALID_ARG;
  // packed RGB with alpha: the alpha byte's shift in the little-endian pixel word (blend.h:55-66: rgba uses the bgra
  // kernels, abgr the argb ones); planar / semi-planar YUV: -1, b200_comp_blend_yuv
  const b200::VideoFormatDesc *d = b200::video_format (out_format);
  int shift;
  if (d && d->family == b200::FAMILY_RGB && d->alpha) shift = 8 * d->pos[0];
  else if (d && (d->family == b200::FAMILY_YUV420 || d->family == b200::FAMILY_NV || d->family == b200::FAMILY_YUV_PLANAR)) shift = -1;
  else return B200_ERR_UNSUPPORTED;
  if (device >= 0) {
    int n = b200_device_count ();
    if (n <= 0) return n < 0 ? n : B200_ERR_NO_DEVICE;
    if (device >= n) return B200_ERR_INVALID_ARG;
  }
  b200_comp *h = new (std::nothrow) b200_comp ();
  if (!h) return B200_ERR_NOMEM;
  h->format = out_format; h->width = width; h->height = height; h->device = device; h->alpha_shift = shift;
  *handle = h;
  return B200_OK;
}

void b200_comp_destroy (b200_comp * h)
{
  if (!h) return;
  if (h->device >= 0) {
    DeviceGuard g (h->device);
    h->ring.drain ();
    h->ring.release ();
    if (h->d_conv) cudaFree (h->d_conv);
  }
  delete h;
}

int b200_comp_blend (b200_comp * h, void *dst, int32_t dst_stride, int background,
    const b200_comp_pad * pads, int n_pads, void *cuda_stream)
{
  if (!h || !dst || n_pads < 0 || n_pads > B200_COMP_MAX_PADS || (n_pads && !pads)) return B200_ERR_INVALID_ARG;
  if (background < 0 || background > 3) return B200_ERR_INVALID_ARG;
  if (h->alpha_shift < 0) return B200_ERR_STATE;                   // created for a 4:2:0 format
  if (dst_stride < h->width * 4 || (dst_stride & 3)) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  CompParams P;
  memset (&P, 0, sizeof (P));
  P.dst = (uint8_t *) dst; P.width = h->width; P.height = h->height; P.stride = dst_stride;
  P.alpha_shift = h->alpha_shift; P.background = background;
  const dim3 grid ((h->width + CT_W - 1) / CT_W, (h->height + CT_H - 1) / CT_H);
  int launched = 0;
  auto flush = [&] () -> int {
    comp_kernel <<<grid, 256, 0, (cudaStream_t) cuda_stream>>> (P);
    B200_CUDA_TRY (cudaGetLastError ());
    launched++;
    P.n_pads = 0; P.background = -1; P.need_recip = 0;
    return B200_OK;
  };
  for (int i = 0; i < n_pads; i++) {
    const b200_comp_pad & pad = pads[i];
    if (!pad.data || pad.width < 1 || pad.height < 1 || pad.stride < pad.width * 4 || (pad.stride & 3))
      return B200_ERR_INVALID_ARG;
    // s_alpha = CLAMP ((gint) (alpha * 255), 0, 255); fully transparent pads are skipped (blend.c:63-67)
    int s_alpha = (int) (pad.alpha * 255);
    s_alpha = s_alpha < 0 ? 0 : (s_alpha > 255 ? 255 : s_alpha);
    if (s_alpha == 0) continue;
    CompPadDev d;
    d.x0 = pad.xpos < 0 ? 0 : pad.xpos; d.y0 = pad.ypos < 0 ? 0 : pad.ypos;
    d.x1 = pad.xpos + pad.width > h->width ? h->width : pad.xpos + pad.width;
    d.y1 = pad.ypos + pad.height > h->height ? h->height : pad.ypos + pad.height;
    if (d.x1 <= d.x0 || d.y1 <= d.y0) continue;
    d.stride = pad.stride;
    d.data = (const uint8_t *) pad.data - (long long) pad.ypos * pad.stride - (long long) pad.xpos * 4;
    d.s_alpha = s_alpha;
    switch (pad.op) {            // blend.c:99-159 with compositor.c:1622-1674 choosing the family
      case B200_COMP_OP_SOURCE: d.mode = s_alpha == 255 ? CM_COPY : CM_SOURCE; break;
      case B200_COMP_OP_OVER: d.mode = background == B200_COMP_BG_TRANSPARENT ? CM_OVERLAY : CM_BLEND; break;
      case B200_COMP_OP_ADD: d.mode = background == B200_COMP_BG_TRANSPARENT ? CM_OVERLAY_ADD : CM_BLEND; break;
      default: return B200_ERR_INVALID_ARG;
    }
    if (d.mode == CM_OVERLAY || d.mode == CM_OVERLAY_ADD) P.need_recip = 1;
    P.pads[P.n_pads++] = d;
    if (P.n_pads == COMP_CHUNK) { int st = flush (); if (st != B200_OK) return st; }
  }
  if (P.n_pads > 0 || launched == 0) { int st = flush (); if (st != B200_OK) return st; }
  return B200_OK;
}

int b200_comp_blend_yuv (b200_comp * h, void *dst, const b200_video_info * di, int background,
    const b200_comp_pad_yuv * pads, int n_pads, void *cuda_stream)
{
  if (!h || !dst || !di || n_pads < 0 || n_pads > B200_COMP_MAX_PADS || (n_pads && !pads)) return B200_ERR_INVALID_ARG;
  if (background < 0 || background > 3) return B200_ERR_INVALID_ARG;
  if (h->alpha_shift >= 0) return B200_ERR_STATE;                  // created for a packed RGB format
  if (di->format != h->format || di->width != h->width || di->height != h->height) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  YuvBlend B;
  int st = B.init (h, dst, di, background, (cudaStream_t) cuda_stream);
  if (st != B200_OK) return st;
  for (int i = 0; i < n_pads; i++) {
    const b200_comp_pad_yuv & pad = pads[i];
    if (pad.info.format != h->format || pad.info.width < 1 || pad.info.height < 1 || !pad.data) return B200_ERR_INVALID_ARG;
    if ((st = B.add (pad.data, pad.info, pad.xpos, pad.ypos, pad.alpha, pad.op)) != B200_OK) return st;
  }
  return B.finish ();
}
int b200_comp_blend_convert (b200_comp * h, void *dst, const b200_video_info * di, int background,
    const b200_comp_pad_convert * pads, int n_pads, void *cuda_stream)
{
  if (!h || !dst || !di || n_pads < 0 || n_pads > B200_COMP_MAX_PADS || (n_pads && !pads)) return B200_ERR_INVALID_ARG;
  if (background < 0 || background > 3) return B200_ERR_INVALID_ARG;
  if (di->format != h->format || di->width != h->width || di->height != h->height) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  const cudaStream_t stream = (cudaStream_t) cuda_stream;
  const bool rgb = h->alpha_shift >= 0;
  const b200::VideoFormatDesc & fd = *b200::video_format (h->format);
  const bool yuv420 = !rgb && (fd.family == b200::FAMILY_YUV420 || fd.family == b200::FAMILY_NV) && fd.bytes == 1;
  int st;
  YuvBlend B;
  if (!rgb && (st = B.init (h, dst, di, background, stream)) != B200_OK) return st;

  // every pad's route; the two-pass pads' converted frames one after another in d_conv (256-byte aligned)
  PadRoute route[B200_COMP_MAX_PADS];
  int xr[B200_COMP_MAX_PADS], yr[B200_COMP_MAX_PADS], rect[B200_COMP_MAX_PADS][4], alpha[B200_COMP_MAX_PADS];
  size_t off[B200_COMP_MAX_PADS], need = 0;
  for (int i = 0; i < n_pads; i++) {
    const b200_comp_pad_convert & pad = pads[i];
    const b200_video_info & in = pad.info;
    if (!pad.data || in.width < 1 || in.height < 1) return B200_ERR_INVALID_ARG;
    if (pad.conv) {
      const b200_video_info & ci = b200::vcs_in_info (pad.conv);
      if (b200::vcs_device (pad.conv) != h->device || b200::vcs_out_info (pad.conv).format != h->format || ci.format != in.format || ci.width != in.width ||
          ci.height != in.height || memcmp (ci.stride, in.stride, sizeof (in.stride)) || memcmp (ci.offset, in.offset, sizeof (in.offset)))
        return B200_ERR_INVALID_ARG;
    } else if (in.format != h->format) {
      return B200_ERR_INVALID_ARG;
    }
    const b200_video_info & fi = pad.conv ? b200::vcs_out_info (pad.conv) : in;     // the frame the blend sees
    bool visible;
    if (rgb) {
      // s_alpha = CLAMP ((gint) (alpha * 255), 0, 255), as b200_comp_blend
      const int a = (int) (pad.alpha * 255);
      alpha[i] = a < 0 ? 0 : (a > 255 ? 255 : a);
      visible = pad.xpos < h->width && pad.ypos < h->height && pad.xpos + fi.width > 0 && pad.ypos + fi.height > 0;
    } else {
      alpha[i] = B.pad_alpha (pad.alpha, pad.op);
      visible = B.place (pad.xpos, pad.ypos, fi.width, fi.height, &xr[i], &yr[i], &rect[i][0], &rect[i][1], &rect[i][2], &rect[i][3]);
    }
    route[i] = pad_route (pad.conv, yuv420, alpha[i], visible);
    if (route[i] == PR_TWO_PASS) {
      off[i] = need;
      need += (b200_video_info_size (&fi) + 255) & ~(size_t) 255;
    }
  }
  if (need > h->conv_cap) {
    B200_CUDA_TRY (cudaFree (h->d_conv));                           // synchronises with blends still reading it
    h->d_conv = nullptr; h->conv_cap = 0;
    B200_CUDA_TRY (cudaMalloc ((void **) &h->d_conv, need));
    h->conv_cap = need;
  }
  // two-pass pads: one batch per converter
  bool done[B200_COMP_MAX_PADS] = {false};
  for (int i = 0; i < n_pads; i++) {
    if (route[i] != PR_TWO_PASS || done[i]) continue;
    const void *in[B200_COMP_MAX_PADS];
    void *out[B200_COMP_MAX_PADS];
    int n = 0;
    for (int j = i; j < n_pads; j++)
      if (route[j] == PR_TWO_PASS && pads[j].conv == pads[i].conv) {
        in[n] = pads[j].data; out[n] = h->d_conv + off[j]; n++;
        done[j] = true;
      }
    if ((st = b200_vcs_convert_batch (pads[i].conv, n, in, out, cuda_stream)) != B200_OK) return st;
  }
  auto blend_data = [&] (int i) -> const uint8_t * {
    return route[i] == PR_TWO_PASS ? h->d_conv + off[i] : (const uint8_t *) pads[i].data;
  };
  auto blend_info = [&] (int i) -> const b200_video_info & {
    return pads[i].conv ? b200::vcs_out_info (pads[i].conv) : pads[i].info;
  };

  if (rgb) {
    b200_comp_pad cp[B200_COMP_MAX_PADS];
    int n = 0;
    for (int i = 0; i < n_pads; i++) {
      if (route[i] == PR_SKIP) continue;
      const b200_video_info & fi = blend_info (i);
      b200_comp_pad & c = cp[n++];
      c.data = blend_data (i) + fi.offset[0];
      c.width = fi.width; c.height = fi.height; c.stride = fi.stride[0];
      c.xpos = pads[i].xpos; c.ypos = pads[i].ypos; c.alpha = pads[i].alpha; c.op = pads[i].op; c.reserved = 0;
    }
    return b200_comp_blend (h, (uint8_t *) dst + di->offset[0], di->stride[0], background, cp, n, cuda_stream);
  }

  // 4:2:0 and the other planar outputs: z-order runs.  A run of blend-kernel pads is one comp_yuv_kernel launch (per
  // CY_MAX_PADS), a run of fused pads one plane-scaler launch per group: pads of one converter that overlap no pad of
  // their own group or of a group launched after it
  int groups = 0, gconv_first[B200_COMP_MAX_PADS], gn[B200_COMP_MAX_PADS], gpad[B200_COMP_MAX_PADS][B200_COMP_MAX_PADS];
  auto overlap = [&] (int a, int b) {
    return rect[a][0] < rect[b][2] && rect[b][0] < rect[a][2] && rect[a][1] < rect[b][3] && rect[b][1] < rect[a][3];
  };
  auto flush_fused = [&] () -> int {
    for (int k = 0; k < groups; k++) {
      CompStore S;
      const uint8_t *in[B200_VCS_MAX_BATCH];
      for (int p = 0; p < 3; p++) { S.dw[p] = B.P.wbytes[p]; S.dh[p] = B.P.rows[p]; }
      for (int j = 0; j < gn[k]; j++) {
        const int i = gpad[k][j];
        in[j] = (const uint8_t *) pads[i].data;
        S.alpha[j] = alpha[i] == CY_COPY ? 256 : alpha[i];
        S.px[0][j] = xr[i]; S.py[0][j] = yr[i];
        for (int p = 1; p < 3; p++) { S.px[p][j] = (xr[i] >> 1) * (B.semi ? 2 : 1); S.py[p][j] = yr[i] >> 1; }
      }
      const int s = b200::vcs_comp_launch (pads[gconv_first[k]].conv, gn[k], in, (uint8_t *) dst, *di, S, stream);
      if (s != B200_OK) return s;
    }
    groups = 0;
    return B200_OK;
  };
  for (int i = 0; i < n_pads; i++) {
    if (route[i] == PR_SKIP) continue;
    if (route[i] != PR_FUSED) {
      if ((st = flush_fused ()) != B200_OK) return st;
      if ((st = B.add (blend_data (i), blend_info (i), pads[i].xpos, pads[i].ypos, pads[i].alpha, pads[i].op)) != B200_OK) return st;
      continue;
    }
    if (B.P.n_pads > 0 || B.launched == 0)                         // what lies below: the background, the blend run
      if ((st = B.finish ()) != B200_OK) return st;
    int g = groups - 1;
    while (g >= 0 && pads[gconv_first[g]].conv != pads[i].conv) g--;
    for (int k = g; g >= 0 && k < groups; k++)
      for (int j = 0; j < gn[k]; j++)
        if (overlap (i, gpad[k][j])) { g = -1; break; }
    if (g < 0) { g = groups++; gconv_first[g] = i; gn[g] = 0; }
    gpad[g][gn[g]++] = i;
  }
  if ((st = flush_fused ()) != B200_OK) return st;
  return B.finish ();
}

int b200_comp_blend_host_submit (b200_comp * h, void *dst_host, int32_t dst_stride, int background,
    const b200_comp_pad * pads, int n_pads)
{
  if (!h || !dst_host || n_pads < 0 || n_pads > B200_COMP_MAX_PADS || (n_pads && !pads)) return B200_ERR_INVALID_ARG;
  if (h->alpha_shift < 0) return B200_ERR_STATE;
  if (dst_stride < h->width * 4 || (dst_stride & 3)) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  B200_CUDA_TRY (h->ring.setup ());
  // staged layout: rows at the caller's stride
  size_t bytes[B200_COMP_MAX_PADS];
  bool up[B200_COMP_MAX_PADS];
  for (int i = 0; i < n_pads; i++) {
    if (!pads[i].data || pads[i].width < 1 || pads[i].height < 1 || pads[i].stride < pads[i].width * 4) return B200_ERR_INVALID_ARG;
    bytes[i] = (size_t) pads[i].stride * pads[i].height;
    up[i] = !(pads[i].alpha <= 0.0 && pads[i].op != B200_COMP_OP_SOURCE);       // else never read by the blend
  }
  return comp_host_submit (h, dst_host, (size_t) dst_stride * h->height, false, pads, n_pads, bytes, up,
      [&] (uint8_t *dst, const b200_comp_pad *dev_pads, cudaStream_t s) {
        return b200_comp_blend (h, dst, dst_stride, background, dev_pads, n_pads, s);
      });
}

int b200_comp_blend_host_wait (b200_comp * h, int keep_in_flight)
{
  if (!h || keep_in_flight < 0) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  if (h->ring.idle (keep_in_flight)) return B200_OK;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  if (keep_in_flight >= b200_comp::kSlots) return B200_ERR_INVALID_ARG;
  B200_CUDA_TRY (h->ring.wait (keep_in_flight));
  return B200_OK;
}

int b200_comp_blend_host (b200_comp * h, void *dst_host, int32_t dst_stride, int background,
    const b200_comp_pad * pads, int n_pads)
{
  int st = b200_comp_blend_host_submit (h, dst_host, dst_stride, background, pads, n_pads);
  if (st != B200_OK) return st;
  return b200_comp_blend_host_wait (h, 0);
}

// planar / semi-planar YUV output from host memory: the same ring of device slots and streams as b200_comp_blend_host_submit;
// every pad frame and the destination travel as whole frames (b200_video_info_size bytes, the caller's plane layout)
int b200_comp_blend_yuv_host_submit (b200_comp * h, void *dst_host, const b200_video_info * di, int background,
    const b200_comp_pad_yuv * pads, int n_pads)
{
  if (!h || !dst_host || !di || n_pads < 0 || n_pads > B200_COMP_MAX_PADS || (n_pads && !pads)) return B200_ERR_INVALID_ARG;
  if (h->alpha_shift >= 0) return B200_ERR_STATE;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  B200_CUDA_TRY (h->ring.setup ());
  size_t bytes[B200_COMP_MAX_PADS];
  bool up[B200_COMP_MAX_PADS];
  for (int i = 0; i < n_pads; i++) {
    if (!pads[i].data || pads[i].info.width < 1 || pads[i].info.height < 1) return B200_ERR_INVALID_ARG;
    bytes[i] = b200_video_info_size (&pads[i].info);
    up[i] = !(pads[i].alpha == 0.0 && pads[i].op != B200_COMP_OP_SOURCE);       // else never read by the blend
  }
  // the blend writes the visible bytes of every plane row only; the rows' stride padding must come back as the caller had it
  // (the reference never touches it), so the destination travels up first
  return comp_host_submit (h, dst_host, b200_video_info_size (di), true, pads, n_pads, bytes, up,
      [&] (uint8_t *dst, const b200_comp_pad_yuv *dev_pads, cudaStream_t s) {
        return b200_comp_blend_yuv (h, dst, di, background, dev_pads, n_pads, s);
      });
}

int b200_comp_blend_yuv_host (b200_comp * h, void *dst_host, const b200_video_info * di, int background,
    const b200_comp_pad_yuv * pads, int n_pads)
{
  int st = b200_comp_blend_yuv_host_submit (h, dst_host, di, background, pads, n_pads);
  if (st != B200_OK) return st;
  return b200_comp_blend_host_wait (h, 0);
}

}  // extern "C"
