// gstreamer_b200/csrc/vcs_device.h — device-side view of a convert+scale plan (product code).
#pragma once

#include <cuda_runtime.h>
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

// How the plane-scaling kernels (vcs_planes*.cuh) store an output byte.  NoStore: into the converter's own output frame.
// CompStore: the compositor's fused route (b200_comp_blend_convert) - item i of the batch is one pad, output byte (x, y)
// of the launch's plane k goes to byte (x + px[k][i], y + py[k][i]) of the compositor's destination plane, is dropped
// outside that plane, and is blended like compositor_orc_blend_u8: (d * (256 - a) + s * a) >> 8, or stored at a >= 256.
struct NoStore { static constexpr bool fused = false; };

struct CompStore {
  static constexpr bool fused = true;
  int dw[3], dh[3];                              // destination plane of the launch's plane k: bytes per row, rows
  int px[3][B200_VCS_MAX_BATCH], py[3][B200_VCS_MAX_BATCH];
  int alpha[B200_VCS_MAX_BATCH];
};

// b200_comp_blend_convert's two halves of the converter (vcs.cu): a converter whose plan is plane scaling into a 4:2:0
// format can store straight into the compositor's destination; vcs_comp_launch runs its plane kernels in their CompStore
// form for n pads (S indexed by destination plane), frames in[i], destination `dst` laid out as `di`
bool vcs_comp_fusable (const b200_vcs * h);
int vcs_device (const b200_vcs * h);
const b200_video_info & vcs_in_info (const b200_vcs * h);
const b200_video_info & vcs_out_info (const b200_vcs * h);
int vcs_comp_launch (b200_vcs * h, int n, const uint8_t *const *in, uint8_t * dst, const b200_video_info & di,
    const CompStore & S, cudaStream_t stream);

}  // namespace b200
