// gstreamer_b200/csrc/vcs_device.h — device-side view of a convert+scale plan (product code).
#pragma once

#include <stdint.h>

#include "../../include/b200dsp.h"

namespace b200 {

struct AxisDev {
  const uint32_t *offset;        // [out_size]
  const int16_t *coef;           // [out_size * coef_per_out]
  const int16_t *sum;            // [out_size] (NTAP only)
  int mode, n_taps, coef_per_out, span, out_size, in_size;
};

// kernel parameter block: plain data, < 4 KB with the batch pointer table
struct VcsDev {
  int iw, ih, ow, oh;
  int stride_y, stride_c, stride_out;
  unsigned long long off_y, off_c, off_out;
  int u_index, h_cosited, v_pairs;
  // chroma components as two strided byte streams: U sample k of chroma row r at in[off_u + r * stride_u + k * cstep]
  // (cstep 2 for the interleaved NV12/NV21 plane, 1 for the I420/YV12 planes)
  unsigned long long off_u, off_v;
  int stride_u, stride_v, cstep;
  int planar;                    // I420 / YV12
  // generic kernel only: bytes between consecutive luma samples (2 in YUY2 / UYVY / YVYU), chroma sub-sampling shifts
  // (horizontal 1 except 4:4:4, vertical 1 only for 4:2:0)
  int ystep, chshift, cvshift;
  int chroma_nearest;            // unchanged-size I420/YV12: the reference's fast path replicates chroma (no filter)
  int h_first, matrix_first;
  int yuv_out;                   // 4:2:0 output through the chain: no matrix stage, scaled A,Y,U,V pixels go to a scratch image
  // packed RGB input (generic kernel only): 4-byte pixels at off_y / stride_y, byte i of (R,G,B) at in_sel nibble i;
  // m = the x256 RGB -> YUV matrix of video_converter_matrix8_table (rows Y,U,V; columns R,G,B,offset)
  int rgb_in;
  unsigned in_sel;
  int m[3][4];
  int p1, p2, p3, p4, p5;
  unsigned sel;                  // byte selector nibbles for PRMT-style packing: byte i <- comp sel[i]
  AxisDev h, v;
  const uint8_t *chroma_mode;    // [ih]
  int tile_w, tile_h, max_rows, cols_pitch, max_crows;
  // planar RGB output (the kernels' planar store form): byte k of the packed pixel goes to plane k
  unsigned long long off_pl[3];
  int stride_pl[3];
};

struct VcsBatch {
  const uint8_t *in[B200_VCS_MAX_BATCH];
  uint8_t *out[B200_VCS_MAX_BATCH];
};

}  // namespace b200
