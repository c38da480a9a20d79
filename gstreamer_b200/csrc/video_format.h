// gstreamer_b200/csrc/video_format.h — what each b200_video_format is: one descriptor per format (host code only).
//
// Header-only: the table and its helpers are inline, so every translation unit that reads a format includes this and
// nothing else needs to be compiled or linked for it.
//
// The converter's plan builder (vcs_plan.cpp), its border fill (vcs.cu), the compositor (comp.cu) and the video-info
// helpers (b200_video_info_set_format / _size) read a format's family, planes, sub-sampling, sample size and component
// positions from here instead of comparing format values.  The facts are GStreamer's format descriptions
// (the formats[] table, gst-libs/gst/video/video-format.c:8184-).
#pragma once

#include "../../include/b200dsp.h"

namespace b200 {

enum FormatFamily : int {
  FAMILY_RGB,                    // packed 4-byte RGB with alpha or padding: RGBx ... ABGR
  FAMILY_RGBP,                   // planar RGB: RGBP, BGRP
  FAMILY_YUV420,                 // planar 4:2:0: I420, YV12, I420_10LE, I420_12LE
  FAMILY_NV,                     // semi-planar 4:2:0: NV12, NV21
  FAMILY_YUV422_PACKED,          // packed 4:2:2: YUY2, UYVY, YVYU
  FAMILY_YUV_PLANAR,             // planar 4:2:2 / 4:4:4: Y42B, Y444 and their 10 / 12 / 16-bit forms
};

struct VideoFormatDesc {
  int format;                    // b200_video_format
  FormatFamily family;
  int n_planes;
  int plane_u, plane_v;          // YUV: the plane holding U / V
  int u_index;                   // semi-planar: byte of U within an interleaved U / V pair
  int wsub, hsub;                // chroma sub-sampling: log2 of the horizontal / vertical factor
  int bytes, depth;              // bytes per sample, bits per sample
  int pair_y, pair_u, pair_v;    // packed 4:2:2: byte of the first Y, of U and of V within a 4-byte pixel pair
  // RGB: the memory byte (packed) or plane (planar) of A, R, G, B.  A format's padding byte stands for A.  Planar RGB
  // has no A plane: A takes byte 3, the byte order of RGBx / BGRx in which the kernels stage planar RGB pixels.
  int pos[4];
  bool alpha;                    // packed RGB: A is alpha, not padding
};

#define F(x) B200_VIDEO_FORMAT_##x
inline constexpr VideoFormatDesc kFormats[] = {
  // format     family                 planes U  V  U-byte ws hs bytes depth  pair Y U V    A  R  G  B   alpha
  {F(RGBx),      FAMILY_RGB,            1,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {3, 0, 1, 2}, false},
  {F(BGRx),      FAMILY_RGB,            1,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {3, 2, 1, 0}, false},
  {F(xRGB),      FAMILY_RGB,            1,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {0, 1, 2, 3}, false},
  {F(xBGR),      FAMILY_RGB,            1,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {0, 3, 2, 1}, false},
  {F(RGBA),      FAMILY_RGB,            1,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {3, 0, 1, 2}, true},
  {F(BGRA),      FAMILY_RGB,            1,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {3, 2, 1, 0}, true},
  {F(ARGB),      FAMILY_RGB,            1,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {0, 1, 2, 3}, true},
  {F(ABGR),      FAMILY_RGB,            1,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {0, 3, 2, 1}, true},
  {F(RGBP),      FAMILY_RGBP,           3,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {3, 0, 1, 2}, false},
  {F(BGRP),      FAMILY_RGBP,           3,     0, 0, 0,     0, 0, 1, 8,       0, 0, 0,    {3, 2, 1, 0}, false},
  {F(I420),      FAMILY_YUV420,         3,     1, 2, 0,     1, 1, 1, 8,       0, 0, 0,    {0, 0, 0, 0}, false},
  {F(YV12),      FAMILY_YUV420,         3,     2, 1, 0,     1, 1, 1, 8,       0, 0, 0,    {0, 0, 0, 0}, false},
  {F(I420_10LE), FAMILY_YUV420,         3,     1, 2, 0,     1, 1, 2, 10,      0, 0, 0,    {0, 0, 0, 0}, false},
  {F(I420_12LE), FAMILY_YUV420,         3,     1, 2, 0,     1, 1, 2, 12,      0, 0, 0,    {0, 0, 0, 0}, false},
  {F(NV12),      FAMILY_NV,             2,     1, 1, 0,     1, 1, 1, 8,       0, 0, 0,    {0, 0, 0, 0}, false},
  {F(NV21),      FAMILY_NV,             2,     1, 1, 1,     1, 1, 1, 8,       0, 0, 0,    {0, 0, 0, 0}, false},
  {F(YUY2),      FAMILY_YUV422_PACKED,  1,     0, 0, 0,     1, 0, 1, 8,       0, 1, 3,    {0, 0, 0, 0}, false},
  {F(UYVY),      FAMILY_YUV422_PACKED,  1,     0, 0, 0,     1, 0, 1, 8,       1, 0, 2,    {0, 0, 0, 0}, false},
  {F(YVYU),      FAMILY_YUV422_PACKED,  1,     0, 0, 0,     1, 0, 1, 8,       0, 3, 1,    {0, 0, 0, 0}, false},
  {F(Y42B),      FAMILY_YUV_PLANAR,     3,     1, 2, 0,     1, 0, 1, 8,       0, 0, 0,    {0, 0, 0, 0}, false},
  {F(Y444),      FAMILY_YUV_PLANAR,     3,     1, 2, 0,     0, 0, 1, 8,       0, 0, 0,    {0, 0, 0, 0}, false},
  {F(I422_10LE), FAMILY_YUV_PLANAR,     3,     1, 2, 0,     1, 0, 2, 10,      0, 0, 0,    {0, 0, 0, 0}, false},
  {F(I422_12LE), FAMILY_YUV_PLANAR,     3,     1, 2, 0,     1, 0, 2, 12,      0, 0, 0,    {0, 0, 0, 0}, false},
  {F(Y444_10LE), FAMILY_YUV_PLANAR,     3,     1, 2, 0,     0, 0, 2, 10,      0, 0, 0,    {0, 0, 0, 0}, false},
  {F(Y444_12LE), FAMILY_YUV_PLANAR,     3,     1, 2, 0,     0, 0, 2, 12,      0, 0, 0,    {0, 0, 0, 0}, false},
  {F(Y444_16LE), FAMILY_YUV_PLANAR,     3,     1, 2, 0,     0, 0, 2, 16,      0, 0, 0,    {0, 0, 0, 0}, false},
};
#undef F

// the descriptor of a format, nullptr for a value the library does not know
inline const VideoFormatDesc * video_format (int format)
{
  for (const VideoFormatDesc & d : kFormats)
    if (d.format == format) return &d;
  return nullptr;
}

// caps defaults (video-info.c:165-185, :211-225) of a format at a frame height: RGB names the RGB matrix and full range
// and leaves the chroma site open; YUV takes BT.709 and H-cosited siting above 576 lines, BT.601 and no siting
// otherwise, and 16-235
struct Colorimetry { int matrix, range, site; };
inline Colorimetry default_colorimetry (const VideoFormatDesc & d, int height)
{
  if (d.family == FAMILY_RGB || d.family == FAMILY_RGBP) return {B200_COLOR_MATRIX_RGB, B200_COLOR_RANGE_0_255, 0};
  const bool hd = height > 576;
  return {hd ? B200_COLOR_MATRIX_BT709 : B200_COLOR_MATRIX_BT601, B200_COLOR_RANGE_16_235,
          hd ? B200_CHROMA_SITE_H_COSITED : B200_CHROMA_SITE_NONE};
}

// fills each unset (0) colour matrix, range and chroma site of *vi with default_colorimetry (d, height)
inline void fill_colorimetry (b200_video_info * vi, const VideoFormatDesc & d, int height)
{
  const Colorimetry c = default_colorimetry (d, height);
  if (vi->color_matrix == 0) vi->color_matrix = c.matrix;
  if (vi->color_range == 0) vi->color_range = c.range;
  if (vi->chroma_site == 0) vi->chroma_site = c.site;
}

// lines per plane of the default layout: 4:2:0 and the 10 / 12-bit 4:2:2 formats round the height up to even
// (video-info.c:997-1009, :1053-1063, :1142-1169), the 8-bit 4:2:2 and the 4:4:4 formats do not (:1020-1041, :1170-1188)
inline int luma_rows (const VideoFormatDesc & d, int height)
{
  return d.hsub || (d.wsub && d.bytes == 2) ? (height + 1) & ~1 : height;
}

}  // namespace b200
