// gstreamer_b200/csrc/vcs_light.cuh — fused kernel for the element's DEFAULT configuration class
// (product code, sm_90a): 4:2:0 semi-planar -> packed RGB where each axis is either untouched /
// nearest (PASS_COPY) or bilinear (PASS_2TAP), horizontal pass first.  BASELINE config C1
// (1920x1080 NV12 -> 1280x720 BGRA, method=bilinear) lands here.
//
// Same arithmetic as vcs_generic_kernel, stage by stage (reference chain: unpack_NV12 -> chroma up
// h,v -> video_orc_resample_h_2tap_4u8_lq -> video_orc_resample_v_2tap_u8_lq ->
// video_orc_convert_AYUV_ARGB -> pack; see vcs_kernels.cuh for the per-stage citations), organised
// around packed 4-byte pixels:
//
//  A  a thread owns 4 consecutive pixels of one input line, or of the two lines of a chroma pair:
//     one LDG.32 of luma per line, the chroma words of the two chroma rows involved, byte-SIMD
//     up-sampling shared by the pair, then four pixels per line leave as one STS.128 of {Y,U,V,-}
//     words (or {A,R,G,B} when the matrix runs first)
//  B  horizontal pass: both taps are whole pixels (2 LDS.32); the lerp runs on two 16-bit lanes per
//     register, so 4 IMAD cover all channels:  (a*(256-f) + b*f) >> 8  never exceeds 16 bits
//  C  vertical pass on the same lane trick:  bits 8..15 of s0*(256-p) + s1*p + 128  is exactly the
//     reference's wrapping 16-bit  s0 + (((s1-s0)*p + 128) >> 8)  for p in [0,256];
//     then the mulhi matrix, byte order, one coalesced 4-byte store per thread.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"
#include "vcs_device.h"
#include "vcs_kernels.cuh"
#include "vcs_lanczos2.cuh"      // packed-byte helpers

namespace b200 {

struct LightDev {
  int tw, th, max_rows, cp;      // tile size, shared-memory rows, words per staged input row
  int t_words;                   // words of the intermediate tile (th x cp when vertical runs first, else none)
  int h_first;
  int std_pairs;                 // every input line consumed in order with the standard 4:2:0 pairing: fast stage A
};

constexpr int LIGHT_THREADS = 256;

// {Y,U,V,-} -> {A,R,G,B} word (A = 255): video_orc_convert_AYUV_ARGB on one pixel
__device__ __forceinline__ unsigned light_matrix (unsigned yuv, const VcsDev & P)
{
  if (P.yuv_out) return __byte_perm (yuv, 0x000000ffu, 0x2104);   // 4:2:0 output: no matrix, {A = 255, Y, U, V} for the down-sampler
  yuv ^= 0x00808080u;
  const int wy = prmt_s (yuv, 0x8800u), wu = prmt_s (yuv, 0x9911u), wv = prmt_s (yuv, 0xaa22u);
  const int ty = ((wy * P.p1) >> 16) + 128;
  const int r = ty + ((wv * P.p2) >> 16);
  const int b = ty + ((wu * P.p3) >> 16);
  const int g = ty + ((wu * P.p4) >> 16) + ((wv * P.p5) >> 16);
  return pack_sat2 (r, 255, pack_sat2 (b, g, 0u));
}

// 4 h-upsampled samples of one chroma component for luma columns x..x+3 (x % 4 == 0).
// e = that component's samples {c[k], c[k+1], c[k+2], -} (k = x/2), p = c[k-1] in byte 0.
template <bool COSITED>
__device__ __forceinline__ unsigned light_hup4 (unsigned e, unsigned p)
{
  const unsigned a = __byte_perm (e, 0, 0x1100);                 // c[k] c[k] c[k+1] c[k+1]
  if (COSITED)                                                   // video_chroma_up_h2_cs_u8: odd px = (l + r + 1) >> 1
    return avg_ceil4 (a, __byte_perm (e, 0, 0x2110));
  // video_chroma_up_h2_u8: even px (c[k-1] + 3c[k] + 2) >> 2, odd px (3c[k] + c[k+1] + 2) >> 2
  const unsigned b = __byte_perm (e, p, 0x2014);                 // c[k-1] c[k+1] c[k] c[k+2]
  return avg_ceil4 (a, avg_floor4 (a, b));
}

// lerp of two packed pixels on 16-bit lanes: every byte = (a*wa + b*wb + rnd) >> 8
__device__ __forceinline__ unsigned light_lerp (unsigned a, unsigned b, unsigned wa, unsigned wb, unsigned rnd)
{
  const unsigned ae = a & 0x00ff00ffu, ao = __byte_perm (a, 0, 0x4341);
  const unsigned be = b & 0x00ff00ffu, bo = __byte_perm (b, 0, 0x4341);
  const unsigned re = ae * wa + (be * wb + rnd), ro = ao * wa + (bo * wb + rnd);
  return __byte_perm (re, ro, 0x7351);
}

// ---- stage A, shared by the light and n-tap kernels ---------------------------------------
// Work list: one entry per input line, or per PAIR of lines (2k+1, 2k+2) that share their two
// chroma rows with swapped 3:1 weights (video_chroma_up_v2_u8) — the h up-sampling of both rows
// and the floor average are then computed once for the two lines.
// entry (uint4) = { row | chroma_mode << 16 | pair << 20, byte offset of the luma line, of its own chroma row, of
// the paired chroma row }; ent[cap].x receives the count.  Call with the whole CTA; only warp 0 works.
__device__ __forceinline__ void vcs_unpack_worklist (const VcsDev & P, int ry0, int R, uint4 *ent, int cap)
{
  const int tid = threadIdx.x;
  if (tid < 32) {
    int count = 0;
    for (int b0 = 0; b0 < R; b0 += 32) {
      const int r = b0 + tid, y = ry0 + r;
      int m = 0, mprev = 0, mnext = 0;
      if (r < R && P.v_pairs) {
        m = P.chroma_mode[y];
        if (r > 0) mprev = P.chroma_mode[y - 1];
        if (r + 1 < R) mnext = P.chroma_mode[y + 1];
      }
      const bool second = m == 2 && mprev == 1 && r > 0;         // handled by the entry of line y-1
      const bool pair = m == 1 && mnext == 2;
      const bool keep = r < R && !second;
      const unsigned mask = __ballot_sync (0xffffffffu, keep);
      if (keep) {
        const int oth = m ? ((m == 1 ? min (y + 1, P.ih - 1) : y - 1) >> 1) : (y >> 1);
        ent[count + __popc (mask & ((1u << tid) - 1u))] = make_uint4 ((unsigned) r | (unsigned) m << 16 | (pair ? 1u << 20 : 0u),
            (unsigned) (y * P.stride_y), (unsigned) ((y >> 1) * P.stride_u), (unsigned) (oth * P.stride_u));
      }
      count += __popc (mask);
    }
    if (tid == 0) ent[cap].x = (unsigned) count;
  }
}

// Unpack + chroma up-sample the tile's input region: a thread owns 4 consecutive pixels (columns
// cxa + 4j ..) of one work-list entry.
// LAYOUT 0: packed pixels {Y,U,V,-} (or {A,R,G,B} when MFIRST) at S[row * pitch + column] (pitch in words).
// LAYOUT 1: three byte planes (Y,U,V or R,G,B) of plane_words words, rows of `pitch` words, 4 pixels per word.
// LAYOUT 2: byte planes in groups of 4 rows, the 4 rows of a word column adjacent:
//           word (row r, column word j, channel ch) at (((r >> 2) * 3 + ch) * pitch + j) * 4 + (r & 3).
template <bool MFIRST, bool COSITED, int LAYOUT>
__device__ __forceinline__ void vcs_unpack_stage (const VcsDev & P, const uint8_t *__restrict__ plane_y,
    const uint8_t *__restrict__ in, int cxa, int ng, const uint4 *ent, int n_ent,
    unsigned *S, int pitch, int plane_words)
{
  const int cw2 = ((P.iw + 1) >> 1) * 2;                         // luma columns covered by whole chroma samples
  const unsigned selU = P.u_index ? 0x7531u : 0x6420u, selV = P.u_index ? 0x6420u : 0x7531u;
  const uint8_t *__restrict__ plane_u = in + P.off_u, *__restrict__ plane_v = in + P.off_v;
  const int hmode = P.chroma_nearest ? 2 : (COSITED ? 1 : 0);    // chroma_hup () filter of the scalar edge path
  const int nitems = n_ent * ng;
  const unsigned magic = 0xffffffffu / (unsigned) ng + 1u;       // item / ng == umulhi (item, magic) for item < 65536, ng > 1

  // the chroma fetch differs between interleaved and planar inputs: two instantiations of the loop, one
  // warp-uniform branch (no predicated-off twin of every address computation)
  auto run = [&] (auto planar_tag) {
    constexpr bool PLANAR = decltype (planar_tag)::value;
  struct Item {                                                  // one work item: 4 pixels of a line or of a line pair
    int r, m, j, x;
    bool pair, fast;
    unsigned co, oo;                                             // byte offsets of chroma sample k = x/2 in its own / paired row
    const uint8_t *rowy;
  };
  // everything the fast path reads from HBM: per chroma row the samples {c[k], c[k+1], c[k+2], c[k+3]} of U and of V
  // (one word each) and c[k-1] (byte 0 of the *p words, non-cosited filter only), then the luma words
  struct Raw { unsigned ue, ve, up, vp, uo, vo, uop, vop, y0, y1; };

  auto decode = [&] (int item) {
    Item it;
    const int e = ng > 1 ? (int) __umulhi ((unsigned) item, magic) : item;
    it.j = item - e * ng;
    const uint4 en = ent[e];
    it.r = (int) (en.x & 0xffffu); it.m = (int) (en.x >> 16) & 3; it.pair = (en.x >> 20) != 0;
    it.x = cxa + 4 * it.j;
    const unsigned kb = (unsigned) (it.x >> 1) * (PLANAR ? 1u : 2u);      // stride_u == stride_v on this path
    it.co = en.z + kb;
    it.oo = en.w + kb;
    it.rowy = plane_y + (en.y + (unsigned) it.x);
    it.fast = it.x + 8 <= cw2 && (COSITED || it.x >= 4 || P.chroma_nearest);
    return it;
  };
  auto load_row = [&] (unsigned off, unsigned & ue, unsigned & ve, unsigned & up, unsigned & vp) {
    up = vp = 0;
    if (PLANAR) {                                                 // two aligned 16-bit loads per component
      const unsigned short *pu = (const unsigned short *) (plane_u + off), *pv = (const unsigned short *) (plane_v + off);
      ue = (unsigned) __ldg (pu) | (unsigned) __ldg (pu + 1) << 16;
      ve = (unsigned) __ldg (pv) | (unsigned) __ldg (pv + 1) << 16;
      if (!COSITED && !P.chroma_nearest) { up = (unsigned) __ldg (pu - 1) >> 8; vp = (unsigned) __ldg (pv - 1) >> 8; }
    } else {                                                      // {U,V} pairs: two words, de-interleaved by PRMT
      const unsigned *pc = (const unsigned *) (in + P.off_c + off);
      const unsigned w0 = __ldg (pc), w1 = __ldg (pc + 1);
      ue = __byte_perm (w0, w1, selU); ve = __byte_perm (w0, w1, selV);
      if (!COSITED) {
        const unsigned wp = __ldg (pc - 1) >> 16;                 // {U,V}[k-1] in bytes 0,1
        up = __byte_perm (wp, 0, selU); vp = __byte_perm (wp, 0, selV);
      }
    }
  };
  auto load_raw = [&] (const Item & it) {                        // loads only: issued back to back for two items
    Raw q;
    load_row (it.co, q.ue, q.ve, q.up, q.vp);
    load_row (it.oo, q.uo, q.vo, q.uop, q.vop);
    q.y0 = __ldg ((const unsigned *) it.rowy);
    q.y1 = it.pair ? __ldg ((const unsigned *) (it.rowy + P.stride_y)) : 0u;
    return q;
  };
  auto store_line = [&] (int rr, int j, unsigned yw, unsigned u, unsigned v) {
    unsigned *d = LAYOUT == 2 ? S + ((rr >> 2) * 3 * pitch + j) * 4 + (rr & 3) : S + rr * pitch + j;
    const int cstep = LAYOUT == 2 ? pitch * 4 : plane_words;      // distance between channels
    if (LAYOUT != 0 && !MFIRST) {
      d[0] = yw; d[cstep] = u; d[2 * cstep] = v;
      return;
    }
    // {Y,U,V,-} per pixel
    const unsigned yu01 = __byte_perm (yw, u, 0x5140), yu23 = __byte_perm (yw, u, 0x7362);       // Y0 U0 Y1 U1
    uint4 px;
    px.x = __byte_perm (yu01, v, 0x4410);
    px.y = __byte_perm (yu01, v, 0x5532);
    px.z = __byte_perm (yu23, v, 0x6610);
    px.w = __byte_perm (yu23, v, 0x7732);
    if (MFIRST) {
      px.x = light_matrix (px.x, P); px.y = light_matrix (px.y, P);
      px.z = light_matrix (px.z, P); px.w = light_matrix (px.w, P);
    }
    if (LAYOUT != 0) {                                           // {A,R,G,B} x 4 -> R, G, B words
      const unsigned rg01 = __byte_perm (px.x, px.y, 0x6251), rg23 = __byte_perm (px.z, px.w, 0x6251);
      const unsigned b01 = __byte_perm (px.x, px.y, 0x0073), b23 = __byte_perm (px.z, px.w, 0x0073);
      d[0] = __byte_perm (rg01, rg23, 0x5410);
      d[cstep] = __byte_perm (rg01, rg23, 0x7632);
      d[2 * cstep] = __byte_perm (b01, b23, 0x5410);
    } else {
      *(uint4 *) (S + rr * pitch + 4 * j) = px;
    }
  };
  auto finish_fast = [&] (const Item & it, const Raw & q) {
    unsigned u, v, ub = 0, vb = 0;
    if (P.chroma_nearest) {                                      // replicate: c[k] c[k] c[k+1] c[k+1]
      u = __byte_perm (q.ue, 0, 0x1100); v = __byte_perm (q.ve, 0, 0x1100);
    } else {
      u = light_hup4<COSITED> (q.ue, q.up);
      v = light_hup4<COSITED> (q.ve, q.vp);
      if (it.m) {                                                // FILT_3_1 / FILT_1_3 against the paired row
        const unsigned uo = light_hup4<COSITED> (q.uo, q.uop), vo = light_hup4<COSITED> (q.vo, q.vop);
        const unsigned fu = avg_floor4 (u, uo), fv = avg_floor4 (v, vo);
        u = avg_ceil4 (u, fu); v = avg_ceil4 (v, fv);
        ub = avg_ceil4 (uo, fu); vb = avg_ceil4 (vo, fv);        // the pair's second line: weights swapped
      }
    }
    store_line (it.r, it.j, q.y0, u, v);
    if (it.pair) store_line (it.r + 1, it.j, q.y1, ub, vb);
  };
  auto slow = [&] (const Item & it) {                            // frame edges: scalar, clamps inside chroma_hup
    unsigned u = 0, v = 0, ub = 0, vb = 0;
    const unsigned kb = (unsigned) (it.x >> 1) * (PLANAR ? 1u : 2u);
    const uint8_t *cu = plane_u + (it.co - kb), *cv = plane_v + (it.co - kb);
    const uint8_t *ou = plane_u + (it.oo - kb), *ov = plane_v + (it.oo - kb);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      if (it.x + i < P.iw) {
        const int u0 = chroma_hup (cu, it.x + i, P.iw, hmode, P.cstep);
        const int v0 = chroma_hup (cv, it.x + i, P.iw, hmode, P.cstep);
        int uu = u0, vv = v0;
        if (it.m) {
          const int u1 = chroma_hup (ou, it.x + i, P.iw, hmode, P.cstep);
          const int v1 = chroma_hup (ov, it.x + i, P.iw, hmode, P.cstep);
          uu = (3 * u0 + u1 + 2) >> 2; vv = (3 * v0 + v1 + 2) >> 2;
          ub |= (unsigned) ((3 * u1 + u0 + 2) >> 2) << (8 * i);
          vb |= (unsigned) ((3 * v1 + v0 + 2) >> 2) << (8 * i);
        }
        u |= (unsigned) uu << (8 * i);
        v |= (unsigned) vv << (8 * i);
      }
    }
    store_line (it.r, it.j, __ldg ((const unsigned *) it.rowy), u, v);
    if (it.pair) store_line (it.r + 1, it.j, __ldg ((const unsigned *) (it.rowy + P.stride_y)), ub, vb);
  };

  // two items per trip: when both take the fast path all their loads are in flight before the first
  // byte-SIMD instruction needs one (the stage is latency bound otherwise)
  // (not when the matrix runs here: its registers cost more occupancy than the overlap returns)
  constexpr bool DUAL = !MFIRST;
  const int stride = (int) blockDim.x;
  for (int item = threadIdx.x; item < nitems; item += (DUAL ? 2 : 1) * stride) {
    const Item a = decode (item);
    const bool has_b = DUAL && item + stride < nitems;
    if (has_b) {
      const Item b = decode (item + stride);
      if (a.fast && b.fast) {
        const Raw qa = load_raw (a), qb = load_raw (b);
        finish_fast (a, qa);
        finish_fast (b, qb);
      } else {
        if (a.fast) finish_fast (a, load_raw (a)); else slow (a);
        if (b.fast) finish_fast (b, load_raw (b)); else slow (b);
      }
    } else {
      if (a.fast) finish_fast (a, load_raw (a)); else slow (a);
    }
  }
  };
  if (P.planar) run (std::true_type {}); else run (std::false_type {});
}

// ---- stage A, fast form ----------------------------------------------------------------------------------------------
// Interleaved chroma (NV12 / NV21), co-sited horizontally, every line of the tile consumed in order (standard pairing:
// line 0 alone, then (1,2), (3,4) ... each pair on two chroma rows with swapped 3:1 weights).  No work list, no per-item
// entry: an item is (line pair q, 8 pixels) - four chroma samples of two rows, one LDG.64 each plus the next sample for the
// last odd pixel, two LDG.64 of luma - and leaves as four STS.128 of {Y,U,V,-} pixels.  Frame edges need no other path:
// chroma rows are clamped (line 0 and the last line then see the same row twice and 3c + c reproduces the unfiltered
// sample), the last odd pixel replicates (video_chroma_up_h2_cs_u8, video-chroma.c:687-699), columns left of the tile's
// first staged word or right of the frame are simply not stored.
// LAYOUT as in vcs_unpack_stage (0: packed pixels; 1 / 2: the byte planes of the n-tap kernels, matrix-last only).
template <bool MFIRST, int LAYOUT = 0, bool PLANAR = false>
__device__ __forceinline__ void vcs_unpack_fast_cs_impl (const VcsDev & P, const uint8_t *__restrict__ in, int cxa, int cx1,
    int ry0, int R, unsigned *S, int pitch, int plane_words = 0)
{
  const uint8_t *__restrict__ plane_y = in + P.off_y, *__restrict__ plane_c = in + P.off_c;
  const unsigned selU = P.u_index ? 0x7531u : 0x6420u, selV = P.u_index ? 0x6420u : 0x7531u;
  // {samples 1..3 of this word, the next sample}: byte 0 of a planar next-sample load, or the U / V byte of the next interleaved pair
  const unsigned sel_nu = (!PLANAR && P.u_index) ? 0x5321u : 0x4321u, sel_nv = (!PLANAR && !P.u_index) ? 0x5321u : 0x4321u;
  const int xs = cxa & ~7;                                        // 8-byte aligned loads
  const int n8 = (min (cx1, P.iw) - xs + 7) >> 3;                 // 8-pixel items per line pair
  const int q0 = (ry0 + 1) >> 1, nq = ((ry0 + R) >> 1) - q0 + 1;  // pairs (2q-1, 2q) touching rows ry0 .. ry0+R-1
  const int crows = (P.ih + 1) >> 1, total = nq * n8;
  const unsigned magic = 0xffffffffu / (unsigned) n8 + 1u;
  for (int item = threadIdx.x; item < total; item += blockDim.x) {
    const int qi = n8 > 1 ? (int) __umulhi ((unsigned) item, magic) : item;
    const int j = item - qi * n8, q = q0 + qi;
    const int x = xs + 8 * j;
    const bool right_edge = x + 8 >= P.iw;                        // no chroma sample to the right of this item
    // at the frame's right edge an odd pixel is averaged with its right neighbour only if that pixel is not the last one
    // (x_odd < iw - 1): byte i of the neighbour word is sample i + 1 for i <= lim, else sample i itself
    const int lim = (P.iw - 3 - x) >> 1;
    const unsigned esel = 0x3210u + (lim >= 0 ? 0x1u : 0u) + (lim >= 1 ? 0x10u : 0u) + (lim >= 2 ? 0x100u : 0u);
    const int ra = min (max (q - 1, 0), crows - 1), rb = min (q, crows - 1);
    // chroma rows a, b as de-interleaved words: {U, V} x 4 samples, and the next sample of each for the last odd pixel
    unsigned uea, vea, ueb, veb, una, vna, unb, vnb;
    if (PLANAR) {                                                 // I420 / YV12: separate planes, 32-bit loads (x / 2 is a multiple of 4)
      const uint8_t *ua = in + P.off_u + (size_t) ra * P.stride_u + (x >> 1), *ub = in + P.off_u + (size_t) rb * P.stride_u + (x >> 1);
      const uint8_t *va = in + P.off_v + (size_t) ra * P.stride_v + (x >> 1), *vb = in + P.off_v + (size_t) rb * P.stride_v + (x >> 1);
      uea = __ldg ((const unsigned *) ua); ueb = __ldg ((const unsigned *) ub);
      vea = __ldg ((const unsigned *) va); veb = __ldg ((const unsigned *) vb);
      una = right_edge ? 0u : (unsigned) __ldg (ua + 4); unb = right_edge ? 0u : (unsigned) __ldg (ub + 4);
      vna = right_edge ? 0u : (unsigned) __ldg (va + 4); vnb = right_edge ? 0u : (unsigned) __ldg (vb + 4);
    } else {
      const uint8_t *pa = plane_c + (size_t) ra * P.stride_c + x, *pb = plane_c + (size_t) rb * P.stride_c + x;
      const uint2 ca = __ldg ((const uint2 *) pa), cb = __ldg ((const uint2 *) pb);
      const unsigned na = right_edge ? 0u : (unsigned) __ldg ((const unsigned short *) (pa + 8));
      const unsigned nb = right_edge ? 0u : (unsigned) __ldg ((const unsigned short *) (pb + 8));
      uea = __byte_perm (ca.x, ca.y, selU); vea = __byte_perm (ca.x, ca.y, selV);
      ueb = __byte_perm (cb.x, cb.y, selU); veb = __byte_perm (cb.x, cb.y, selV);
      una = vna = na; unb = vnb = nb;                             // the next pair: its U / V byte is picked by sel_nu / sel_nv
    }
    const int ya = 2 * q - 1, yb = 2 * q;                         // the pair's lines; ya == -1 for q == 0
    const bool sa = ya >= ry0 && ya < ry0 + R, sb = yb >= ry0 && yb < ry0 + R && yb < P.ih;
    uint2 y0 = make_uint2 (0u, 0u), y1 = make_uint2 (0u, 0u);
    if (sa) y0 = __ldg ((const uint2 *) (plane_y + (size_t) ya * P.stride_y + x));
    if (sb) y1 = __ldg ((const uint2 *) (plane_y + (size_t) yb * P.stride_y + x));
    // co-sited h up-sampling of both rows: even pixel = c[k], odd pixel = (c[k] + c[k+1] + 1) >> 1
    unsigned alo[2], ahi[2], blo[2], bhi[2];                      // [U, V] x 8 full-resolution samples (lo = pixels 0..3)
    {
      const unsigned ue = uea, ve = vea;
      const unsigned un = right_edge ? __byte_perm (ue, ue, esel) : __byte_perm (ue, una, sel_nu);
      const unsigned vn = right_edge ? __byte_perm (ve, ve, esel) : __byte_perm (ve, vna, sel_nv);
      const unsigned uo = avg_ceil4 (ue, un), vo = avg_ceil4 (ve, vn);
      alo[0] = __byte_perm (ue, uo, 0x5140); ahi[0] = __byte_perm (ue, uo, 0x7362);
      alo[1] = __byte_perm (ve, vo, 0x5140); ahi[1] = __byte_perm (ve, vo, 0x7362);
    }
    {
      const unsigned ue = ueb, ve = veb;
      const unsigned un = right_edge ? __byte_perm (ue, ue, esel) : __byte_perm (ue, unb, sel_nu);
      const unsigned vn = right_edge ? __byte_perm (ve, ve, esel) : __byte_perm (ve, vnb, sel_nv);
      const unsigned uo = avg_ceil4 (ue, un), vo = avg_ceil4 (ve, vn);
      blo[0] = __byte_perm (ue, uo, 0x5140); bhi[0] = __byte_perm (ue, uo, 0x7362);
      blo[1] = __byte_perm (ve, vo, 0x5140); bhi[1] = __byte_perm (ve, vo, 0x7362);
    }
    // the pair: line 2q-1 = (3a + b + 2) >> 2, line 2q = (a + 3b + 2) >> 2   (video_chroma_up_v2_u8)
    unsigned u0[2], v0[2], u1[2], v1[2];                          // [pixels 0..3, pixels 4..7]
    {
      unsigned f;
      f = avg_floor4 (alo[0], blo[0]); u0[0] = avg_ceil4 (alo[0], f); u1[0] = avg_ceil4 (blo[0], f);
      f = avg_floor4 (ahi[0], bhi[0]); u0[1] = avg_ceil4 (ahi[0], f); u1[1] = avg_ceil4 (bhi[0], f);
      f = avg_floor4 (alo[1], blo[1]); v0[0] = avg_ceil4 (alo[1], f); v1[0] = avg_ceil4 (blo[1], f);
      f = avg_floor4 (ahi[1], bhi[1]); v0[1] = avg_ceil4 (ahi[1], f); v1[1] = avg_ceil4 (bhi[1], f);
    }
    auto store4 = [&] (int row, int col, unsigned yw, unsigned u, unsigned v) {
      if (col < 0 || col + cxa >= cx1) return;                    // left of the tile's first staged word / right of its last column
      if (LAYOUT != 0) {                                          // byte planes: one word of 4 pixels per channel
        const int j = col >> 2;
        unsigned *d = LAYOUT == 2 ? S + ((row >> 2) * 3 * pitch + j) * 4 + (row & 3) : S + row * pitch + j;
        const int cstep = LAYOUT == 2 ? pitch * 4 : plane_words;
        d[0] = yw; d[cstep] = u; d[2 * cstep] = v;
        return;
      }
      const unsigned yu01 = __byte_perm (yw, u, 0x5140), yu23 = __byte_perm (yw, u, 0x7362);
      uint4 px;
      px.x = __byte_perm (yu01, v, 0x4410);
      px.y = __byte_perm (yu01, v, 0x5532);
      px.z = __byte_perm (yu23, v, 0x6610);
      px.w = __byte_perm (yu23, v, 0x7732);
      if (MFIRST) {
        px.x = light_matrix (px.x, P); px.y = light_matrix (px.y, P);
        px.z = light_matrix (px.z, P); px.w = light_matrix (px.w, P);
      }
      *(uint4 *) (S + row * pitch + col) = px;
    };
    const int col = x - cxa;
    if (sa) { store4 (ya - ry0, col, y0.x, u0[0], v0[0]); store4 (ya - ry0, col + 4, y0.y, u0[1], v0[1]); }
    if (sb) { store4 (yb - ry0, col, y1.x, u1[0], v1[0]); store4 (yb - ry0, col + 4, y1.y, u1[1], v1[1]); }
  }
}

// semi-planar (NV12 / NV21) or planar (I420 / YV12) chroma: a property of the plan, two instantiations of the stage
template <bool MFIRST, int LAYOUT = 0>
__device__ __forceinline__ void vcs_unpack_fast_cs (const VcsDev & P, const uint8_t *__restrict__ in, int cxa, int cx1,
    int ry0, int R, unsigned *S, int pitch, int plane_words = 0)
{
  if (P.planar) vcs_unpack_fast_cs_impl<MFIRST, LAYOUT, true> (P, in, cxa, cx1, ry0, R, S, pitch, plane_words);
  else vcs_unpack_fast_cs_impl<MFIRST, LAYOUT, false> (P, in, cxa, cx1, ry0, R, S, pitch, plane_words);
}

// PLOUT: planar RGB output (store_planar_px) instead of one 4-byte word per pixel
template <int HM, int VM, bool MFIRST, bool COSITED, bool PLOUT = false>
__global__ void __launch_bounds__ (LIGHT_THREADS, 4)
vcs_light_kernel (const VcsDev P, const LightDev G, const VcsBatch frames)
{
  extern __shared__ __align__ (16) unsigned lsm[];
  unsigned *S = lsm;                                             // [max_rows][cp]   staged input pixels
  unsigned *T = lsm + G.max_rows * G.cp;                         // [max_rows][tw]   after the h pass
  const int tid = threadIdx.x;
  const uint8_t *__restrict__ in = frames.in[blockIdx.z];
  uint8_t *__restrict__ out = frames.out[blockIdx.z];
  const uint8_t *__restrict__ plane_y = in + P.off_y;

  const int ox0 = blockIdx.x * G.tw, oy0 = blockIdx.y * G.th;
  const int tw = min (G.tw, P.ow - ox0), th = min (G.th, P.oh - oy0);
  const int cx0 = P.h.offset[ox0], cx1 = P.h.offset[ox0 + tw - 1] + P.h.span;
  const int ry0 = P.v.offset[oy0], ry1 = P.v.offset[oy0 + th - 1] + P.v.span;
  const int cxa = cx0 & ~3, R = ry1 - ry0, ng = (cx1 - cxa + 3) >> 2;

  // ---------------------------------------------------------------- A: unpack + chroma up-sample
  uint4 *ent = (uint4 *) (T + G.t_words);                        // [max_rows] entries, then the count
  unsigned *vtab = (unsigned *) (ent + G.max_rows + 1);          // [th] vertical source row and weight of each output row
  if (tid >= 32 && tid < 32 + th) {
    const int oy = oy0 + tid - 32;
    vtab[tid - 32] = (P.v.offset[oy] - (unsigned) ry0) | (VM == 2 ? (unsigned) (int) P.v.coef[oy] << 16 : 0u);
  }
  if (COSITED && G.std_pairs) {                                   // warp-uniform: a property of the plan
    vcs_unpack_fast_cs<MFIRST> (P, in, cxa, cx1, ry0, R, S, G.cp);
  } else {
    vcs_unpack_worklist (P, ry0, R, ent, G.max_rows);
    __syncthreads ();
    vcs_unpack_stage<MFIRST, COSITED, 0> (P, plane_y, in, cxa, ng, ent, (int) ent[G.max_rows].x, S, G.cp, 0);
  }
  __syncthreads ();

  const int tx = tid & 127, rph = tid >> 7;                      // tw <= 128, two row phases
  if (G.h_first) {
    // -------------------------------------------------------------- B + C fused: a thread owns one output column and walks
    // half of the tile's output rows top to bottom.  The h-lerped value of its column is kept in registers for the two
    // source rows of the current output row; the next output row re-uses them when its source rows repeat (always for an
    // up-scale, every other row at 1.5:1) - no intermediate tile, no second barrier.  Rounding is unchanged: the h pass
    // rounds to 8 bits before the v pass sees it (video-scaler.c:609-618, :846-879).
    if (tx < tw) {
      const int base = (int) P.h.offset[ox0 + tx] - cxa;
      unsigned f = 0;
      if (HM == 2) f = (unsigned) (int) P.h.coef[ox0 + tx];
      const unsigned *col = S + base;
      auto hrow = [&] (int r) {
        const unsigned a = col[r * G.cp];
        return HM == 2 ? light_lerp (a, col[r * G.cp + 1], 256u - f, f, 0u) : a;
      };
      // rows in PAIRS without carried state: the pair (ty, ty+1) needs source rows (a0, a0+1) and (a1, a1+1) - three h-lerps
      // when a1 == a0 + 1 (every pair at 1.5:1: rows 3k, 3k+1, 3k+2), two when a1 == a0 (up-scaling), four otherwise.  (The
      // first form carried the last two h-lerped rows from one output row to the next through a three-way branch: 80
      // instructions per output pixel of which 30 were the loop's own.)
      const int half = (((th + 1) >> 1) + 1) & ~1, t0 = rph * half, t1 = min (th, t0 + half);
      uint8_t *dst = out + P.off_out + (size_t) (oy0 + t0) * P.stride_out + (size_t) (ox0 + tx) * 4u;
      auto finish = [&] (unsigned d, uint8_t *q, int ty) {
        if (!MFIRST) d = light_matrix (d, P);
        else d |= 0x000000ffu;                                    // alpha passes every 2-tap/copy stage as 255
        if (PLOUT) store_planar_px (P, out, ox0 + tx, oy0 + ty, __byte_perm (d, 0, P.sel));
        else *(unsigned *) q = __byte_perm (d, 0, P.sel);
      };
      for (int ty = t0; ty < t1; ty += 2, dst += 2 * (size_t) P.stride_out) {
        const bool two = ty + 1 < t1;
        const unsigned vo0 = vtab[ty], vo1 = vtab[two ? ty + 1 : ty];   // row offset inside the tile | weight << 16
        const int a0 = (int) (vo0 & 0xffffu), a1 = (int) (vo1 & 0xffffu);
        unsigned d0, d1;
        if (VM == 2) {
          const unsigned p0 = vo0 >> 16, p1 = vo1 >> 16;
          const unsigned h0 = hrow (a0), h1 = hrow (a0 + 1);
          d0 = light_lerp (h0, h1, 256u - p0, p0, 0x00800080u);
          if (a1 == a0 + 1) {                                     // warp-uniform: every lane has the same output rows
            const unsigned h2 = hrow (a1 + 1);
            d1 = light_lerp (h1, h2, 256u - p1, p1, 0x00800080u);
          } else if (a1 == a0) {
            d1 = light_lerp (h0, h1, 256u - p1, p1, 0x00800080u);
          } else {
            const unsigned h2 = hrow (a1), h3 = hrow (a1 + 1);
            d1 = light_lerp (h2, h3, 256u - p1, p1, 0x00800080u);
          }
        } else {
          d0 = hrow (a0);
          d1 = a1 == a0 ? d0 : hrow (a1);
        }
        finish (d0, dst, ty);
        if (two) finish (d1, dst + P.stride_out, ty + 1);
      }
    }
  } else {
    // vertical pass first (chain_scale when out_w * in_h > in_w * out_h): same two lerps, other order
    const int C = cx1 - cxa, lane = tid & 31;
    for (int ty = tid >> 5; ty < th; ty += LIGHT_THREADS / 32) {
      const unsigned vo = vtab[ty];
      const unsigned *s0 = S + (vo & 0xffffu) * G.cp;
      const unsigned p = vo >> 16;
      for (int c = lane; c < C; c += 32) {
        unsigned d = s0[c];
        if (VM == 2) d = light_lerp (d, s0[G.cp + c], 256u - p, p, 0x00800080u);
        T[ty * G.cp + c] = d;
      }
    }
    __syncthreads ();
    if (tx < tw) {
      const int base = (int) P.h.offset[ox0 + tx] - cxa;
      unsigned f = 0;
      if (HM == 2) f = (unsigned) (int) P.h.coef[ox0 + tx];
      uint8_t *dst = out + P.off_out + (size_t) (oy0 + rph) * P.stride_out + (size_t) (ox0 + tx) * 4u;
      const size_t dstep = (size_t) P.stride_out * (LIGHT_THREADS / 128);
      for (int ty = rph; ty < th; ty += LIGHT_THREADS / 128, dst += dstep) {
        const unsigned *t = T + ty * G.cp + base;
        unsigned d = t[0];
        if (HM == 2) d = light_lerp (d, t[1], 256u - f, f, 0u);
        if (!MFIRST) d = light_matrix (d, P);
        else d |= 0x000000ffu;
        if (PLOUT) store_planar_px (P, out, ox0 + tx, oy0 + ty, __byte_perm (d, 0, P.sel));
        else *(unsigned *) dst = __byte_perm (d, 0, P.sel);
      }
    }
  }
}

typedef void (*light_kernel_fn) (const VcsDev, const LightDev, const VcsBatch);

inline light_kernel_fn light_kernel_for (const VcsPlan & p)
{
#define LIGHT_PICK(HM, VM)                                                                            \
  if (p.h.mode == HM && p.v.mode == VM) {                                                             \
    if (p.rgbp_out) {                                                                                 \
      if (p.matrix_first) return p.h_cosited ? vcs_light_kernel<HM, VM, true, true, true> : vcs_light_kernel<HM, VM, true, false, true>;   \
      return p.h_cosited ? vcs_light_kernel<HM, VM, false, true, true> : vcs_light_kernel<HM, VM, false, false, true>;                     \
    }                                                                                                 \
    if (p.matrix_first) return p.h_cosited ? vcs_light_kernel<HM, VM, true, true> : vcs_light_kernel<HM, VM, true, false>;   \
    return p.h_cosited ? vcs_light_kernel<HM, VM, false, true> : vcs_light_kernel<HM, VM, false, false>;                     \
  }
  LIGHT_PICK (1, 1) LIGHT_PICK (1, 2) LIGHT_PICK (2, 1) LIGHT_PICK (2, 2)
#undef LIGHT_PICK
  return nullptr;
}

inline int launch_light (const VcsDev & dev, const VcsPlan & p, const VcsBatch & batch, int n, cudaStream_t stream)
{
  light_kernel_fn fn = light_kernel_for (p);
  if (!fn) return B200_ERR_STATE;
  LightDev g;
  g.tw = p.light_tw; g.th = p.light_th; g.max_rows = p.light_rows; g.cp = p.light_cp;
  g.h_first = p.h_first ? 1 : 0;
  g.std_pairs = p.light_std_pairs ? 1 : 0;
  for (int i = 0; i < n; i++) if (((uintptr_t) batch.in[i]) & 7) g.std_pairs = 0;     // the fast stage A loads 64 bits at a time
  g.t_words = p.h_first ? 0 : p.light_th * p.light_cp;
  dim3 grid ((p.out.width + g.tw - 1) / g.tw, (p.out.height + g.th - 1) / g.th, n);
  fn <<<grid, LIGHT_THREADS, p.light_smem, stream>>> (dev, g, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

}  // namespace b200
