// gstreamer_b200/csrc/vcs_plan.h — host-side per-caps plan of the convert+scale path.
//
// Product code.  This is the CUDA build's equivalent of the one-time setup the
// reference does in gst_video_converter_new_with_pool()/chain_*()
// (gst-libs/gst/video/video-converter.c:2421, :852-2112): instead of a chain of
// line caches it produces flat tables the fused kernels index directly.
#pragma once

#include <stddef.h>
#include <stdint.h>
#include <functional>
#include <vector>

#include "../../include/b200dsp.h"

namespace b200 {

// pass kinds understood by the kernels
enum PassMode : int { PASS_COPY = 1, PASS_2TAP = 2, PASS_NTAP = 3 };

struct AxisPlan {
  int in_size = 0, out_size = 0;
  int mode = PASS_COPY;          // PASS_COPY covers "no scaling" (identity offsets) and nearest
  int n_taps = 1;                // taps per output sample as the reference counts them
  int coef_per_out = 0;          // int16 coefficients stored per output sample (0, 1 or n_taps)
  int span = 1;                  // input samples read per output sample
  bool scaling = false;
  std::vector<uint32_t> offset;  // first input sample of each output sample
  std::vector<int16_t> coef;     // NTAP: n_taps 6-bit taps; 2TAP-h: 8-bit fraction; 2TAP-v: 8-bit p1
  std::vector<int16_t> sum;      // NTAP: sum of taps (alpha channel), else unused
};

// YUV -> same YUV family (convert_scale_planes, video-converter.c:7757-7769): one of these per output plane
enum PlaneMode : int { PM_COPY = 0, PM_HALVE_V = 1, PM_HALVE_H = 2, PM_HALVE_HV = 3, PM_DOUBLE = 4, PM_SCALE = 5 };
struct PlanePlan {
  int src_plane = 0;             // plane of the input that feeds this output plane
  int iw = 0, ih = 0, ow = 0, oh = 0;    // in pixels of this plane
  int ne = 1;                    // bytes per pixel (2 for the interleaved UV plane, 4 for packed RGB)
  unsigned swz = 0;              // packed RGB to another byte order: output byte c <- source byte (swz >> 4c) & 3
  int mode = PM_COPY;
  bool have_h = false, have_v = false, h_first = true;
  AxisPlan h, v;
};

struct VcsPlan {
  b200_video_info in, out;
  b200_vcs_config cfg;
  AxisPlan h, v;
  bool h_first = true;
  bool matrix_first = false;
  int p[5] = {0, 0, 0, 0, 0};
  int im[4][4];
  bool h_cosited = false, v_pairs = true;
  int u_index = 0;               // byte index of U inside an interleaved chroma pair
  bool planar = false;           // I420 / YV12: separate U and V planes
  int plane_u = 1, plane_v = 1;  // plane index holding U / V
  bool chroma_nearest = false;   // planar input at unchanged size: convert_I420_BGRA family fast path
  // 4:2:2 / 4:4:4 inputs (generic kernel only): luma sample pitch, chroma shifts, byte offsets of Y / U / V samples
  int ystep = 1, chshift = 1, cvshift = 1, cstep_in = 0;
  uint64_t in_off_y = 0, in_off_u = 0, in_off_v = 0;
  int in_stride_u = 0, in_stride_v = 0;
  bool in_422_444 = false;
  bool yuy2_420 = false;         // YUY2 / UYVY -> I420 / YV12 at an unchanged size: the reference's table row (vcs_yuy2_420.cuh)
  uint8_t byte_sel[4] = {3, 2, 1, 0};   // output byte i takes component byte_sel[i] of (A,R,G,B)
  std::vector<uint8_t> chroma_mode;     // per input line: 0 own row, 1 first of pair, 2 second

  // generic tiled kernel geometry
  int tile_w = 64, tile_h = 16;
  int max_rows = 0, max_cols = 0, cols_pitch = 0, max_crows = 0;
  int smem_bytes = 0;

  // 4:2:0 output: per-plane scaling instead of the unpack -> ... -> pack chain
  bool planes_mode = false;
  int n_planes = 0;
  PlanePlan planes[3];

  // 4:2:0 -> the other 4:2:0 family (NV12 <-> I420, NV12 <-> NV21 ...): the chain without a matrix stage, then
  // chroma down-sampling + pack (vcs_down420.cuh)
  bool yuv_out = false;
  int down_h = 0;                // Down420H: none / pair average / co-sited 3-1, 1-2-1, 1-3
  bool down_v = false;           // average the line pair (out site not V_COSITED)
  bool extra_row = false;        // odd height, no vertical scaler: the last pair's second line is rebuilt (see build_vcs_plan)
  int out_plane_u = 1, out_plane_v = 1, out_cstep = 1, out_u_index = 0;

  // packed RGB input -> 4:2:0 (generic kernel only): byte selector to (R,G,B,A) and the x256 table matrix
  bool rgb_in = false;
  unsigned in_sel = 0x3210;
  int m_rgb2yuv[3][4] = {{0}};

  // destination rectangle (the element's add-borders): `out` above describes the RECTANGLE (same strides, plane
  // origins shifted to its first pixel) so that every kernel runs unchanged; frame_out is the whole output frame
  bool has_dest = false;
  b200_video_info frame_out;
  int dest[4] = {0, 0, 0, 0};     // x, y, width, height in luma pixels
  bool fill_border = true;
  uint8_t border_px[4] = {0, 0, 0, 0};   // packed RGB outputs: the border pixel in memory order
  int border_yuv[3] = {16, 128, 128};    // 4:2:0 outputs

  // planar RGB output (RGBP / BGRP).  YUV inputs: the packed RGB plan with the byte selector of RGBx / BGRx, so that
  // byte k of each packed pixel is the component of plane k; the kernels' planar store form writes it to
  // out.offset[k] + y * out.stride[k] + x.  Packed RGB inputs: planes[0] scales the 4-byte pixels (input byte order)
  // into a scratch image when the size changes, then a de-interleave launch writes plane k from source byte
  // (deint_sel >> 4k) & 3.
  bool rgbp_out = false;
  unsigned deint_sel = 0;

  // specialised 2:1 lanczos kernel eligibility
  bool lanczos2_ok = false;

  // n-tap kernel (vcs_ntap.cuh): dp4a FIRs on planar tiles, any ratio, horizontal first
  bool ntap_ok = false;
  int ntap_tw = 128, ntap_th = 16, ntap_rows = 0, ntap_pitch = 0, ntap_smem = 0;   // rows: multiple of 4; pitch in words
  int ntw_h = 0, ntw_v = 0;              // packed tap words per output (0 for a copy axis)
  std::vector<int32_t> h_packed, v_packed;
  bool ntap_alpha_opaque = true;

  // "light" kernel (both axes copy or 2-tap, horizontal first): tile geometry
  bool light_ok = false;
  int light_tw = 128, light_th = 16, light_rows = 0, light_cp = 0, light_smem = 0;
  bool light_std_pairs = false;          // standard in-order 4:2:0 pairing, interleaved chroma, 8-byte aligned planes: fast stage A
};

// builds everything that does not need a device; returns b200_status
int build_vcs_plan (const b200_video_info * in, const b200_video_info * out,
    const b200_vcs_config * cfg, VcsPlan * plan);

// What the tiles of one axis stage, `tile` outputs to a tile: the input samples from the first output's window start
// to the last output's window end; on the word grid from a 4-aligned start, the extent rounded up to whole words.
struct StagedExtent {
  int extent = 0;                // the most input samples any tile stages
  int max_base = 0;              // the furthest an output's window starts from its tile's staged start
  bool inside = true;            // every output's window [offset, offset + span) lies inside its tile's staged range
};
StagedExtent staged_extent (const AxisPlan & a, int tile, bool word_grid);

// A tile shape of the dp4a kernels (n-tap, plane scaler): tw x th outputs, the staged lines rounded up to whole 4-line
// groups, the staged columns on the word grid
struct TileShape {
  int tw = 0, th = 0, rows = 0, cols = 0;
  StagedExtent x, y;
  int pitch = 0;                 // words per staged line, set by the kernel's shared-memory formula
  size_t smem = 0;
};
// The shape of `shapes` that stages the fewest input pixels per output pixel, among those whose windows lie inside
// the staged ranges and whose shared memory lets at least two CTAs share an SM.  smem (shape) is the kernel's
// formula: it sets shape.pitch and returns the bytes, 0 for a shape the kernel cannot run.  The environment variable
// `env` ("tw,th", a tuning aid) restricts the search to that shape.  False when no shape qualifies.
bool search_tile_shape (const AxisPlan & h, const AxisPlan & v, const int (*shapes)[2], int n_shapes, const char *env,
    const std::function<size_t (TileShape &)> & smem, TileShape * best);

// 4 signed 8-bit taps per word, zero padded to a whole number of words; false when a tap does not fit or the 16-bit
// accumulator of the reference could wrap (the dp4a kernels accumulate in 32 bits).  ntw = 0 for other than n-tap axes.
bool pack_taps_s8 (const AxisPlan & a, int *ntw, std::vector<int32_t> * out);
// the tap-word count the dp4a kernels take as a template argument: the n-tap axis's, both axes' when they agree, else
// 0 (counted at run time)
int common_tap_words (int h_mode, int v_mode, int ntw_h, int ntw_v);
// an n-tap axis whose every tap sum lies in [64, 128] keeps alpha at 255 (other axes do not touch it)
bool alpha_stays_opaque (const AxisPlan & a);
// every input line pulled in order with the standard 4:2:0 pairing: line 0 alone, then (1, 2), (3, 4) ...
bool standard_pairing (const VcsPlan & p);

}  // namespace b200
