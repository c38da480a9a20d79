/* gst/gstcudavideoconvertscale.c — `cudavideoconvertscale`
 *
 * Drop-in for `videoconvertscale` on CUDA memory: same properties (method, envelope, sharpness,
 * sharpen; gst-plugins-base/gst/videoconvertscale/gstvideoconvertscale.c:306-391), same caps
 * transform rules (:703-748, restricted to the formats libb200dsp implements), and a
 * transform() that hands the mapped device frames to b200_vcs_convert() where the stock
 * element calls gst_video_converter_frame() (:1981-2005).  Device-memory plumbing (context
 * sharing, stream selection, allocation queries) follows the stock CUDA converter
 * gst-plugins-bad/sys/nvcodec/gstcudaconvertscale.c:1483-1587 and gstcudabasetransform.c.
 *
 * NOT built in the development image (no GLib/GStreamer there); `make -C gst/check` runs the sources through
 * gcc -fsyntax-only against declarations restated from the reference headers (gst/check/), see INTEGRATION.md.
 */
#include <gst/base/gstbasetransform.h>
#include <gst/cuda/gstcuda.h>

#include "gstb200elements.h"

GST_DEBUG_CATEGORY_STATIC (cuda_vcs_debug);
#define GST_CAT_DEFAULT cuda_vcs_debug

/* what b200_vcs_create accepts: every sink format to every src format - 4:2:0, packed RGB, packed 4:2:2 (capture) and planar
 * Y42B / Y444 in; packed RGB (scaling, byte order), planar RGB (a network's CHW input) or 4:2:0 (the encoder-feeding
 * direction) out */
#define YUV420_FORMATS "NV12, NV21, I420, YV12"
#define RGB_FORMATS "BGRA, RGBA, ARGB, ABGR, BGRx, RGBx, xRGB, xBGR"
#define PACKED422_FORMATS "YUY2, UYVY, YVYU"
#define PLANAR4XX_FORMATS "Y42B, Y444"
#define PLANAR_RGB_FORMATS "RGBP, BGRP"
#define CAPTURE_FORMATS PACKED422_FORMATS ", " PLANAR4XX_FORMATS
#define SINK_FORMATS "{ " YUV420_FORMATS ", " RGB_FORMATS ", " CAPTURE_FORMATS " }"
/* YUV outputs: the same family (NV12->NV12, NV21->NV21, I420/YV12 -> I420/YV12) scales plane by plane, the other
 * 4:2:0 pairs run the chain with chroma down-sampling; fixate_caps must carry the input colorimetry over
 * (transfer_colorimetry_from_input, gstvideoconvertscale.c:1335-1427) - b200_vcs_create refuses a YUV -> YUV
 * matrix change with B200_ERR_UNSUPPORTED */
#define SRC_FORMATS "{ " RGB_FORMATS ", " PLANAR_RGB_FORMATS ", " YUV420_FORMATS " }"
#define RAW_FIELDS(f) "format = (string) " f \
    ", width = (int) [ 1, 32767 ], height = (int) [ 1, 32767 ], framerate = (fraction) [ 0/1, max ]"
/* device memory first (zero copy between CUDA elements), then plain system memory: in that case transform() hands the
 * mapped host frames to b200_vcs_convert_host(), whose pinned-slot pipeline does the H2D / D2H - the element drops in
 * for videoconvertscale without cudaupload / cudadownload around it */
#define BOTH_CAPS(f) "video/x-raw(" GST_CAPS_FEATURE_MEMORY_CUDA_MEMORY "), " RAW_FIELDS (f) "; video/x-raw, " RAW_FIELDS (f)

static GstStaticPadTemplate sink_tmpl = GST_STATIC_PAD_TEMPLATE ("sink", GST_PAD_SINK, GST_PAD_ALWAYS,
    GST_STATIC_CAPS (BOTH_CAPS (SINK_FORMATS)));
static GstStaticPadTemplate src_tmpl = GST_STATIC_PAD_TEMPLATE ("src", GST_PAD_SRC, GST_PAD_ALWAYS,
    GST_STATIC_CAPS (BOTH_CAPS (SRC_FORMATS)));

enum { PROP_0, PROP_METHOD, PROP_ENVELOPE, PROP_SHARPNESS, PROP_SHARPEN, PROP_ADD_BORDERS, PROP_DEVICE_ID,
  /* the stock element's remaining properties (gstvideoconvertscale.c:326-391): installed so that existing pipelines keep
   * working; only the default of each is implemented (vcs_rebuild refuses anything else), n-threads is free */
  PROP_DITHER, PROP_N_THREADS, PROP_DITHER_QUANTIZATION, PROP_CHROMA_RESAMPLER, PROP_ALPHA_MODE, PROP_ALPHA_VALUE,
  PROP_CHROMA_MODE, PROP_MATRIX_MODE, PROP_GAMMA_MODE, PROP_PRIMARIES_MODE
};

typedef struct
{
  GstBaseTransform parent;
  /* properties (defaults: gstvideoconvertscale.c:130-144) */
  gint method;
  gdouble envelope, sharpness, sharpen;
  gboolean add_borders;           /* DEFAULT_PROP_ADD_BORDERS TRUE, gstvideoconvertscale.c:131 */
  gint device_id;
  gint dither, chroma_resampler, alpha_mode, chroma_mode, matrix_mode, gamma_mode, primaries_mode;
  guint n_threads, dither_quantization;
  gdouble alpha_value;
  gboolean config_changed;
  /* negotiated state */
  GstVideoInfo in_info, out_info;
  GstCudaContext *context;
  GstCudaStream *stream;
  b200_vcs *vcs;
} GstCudaVideoConvertScale;

typedef struct { GstBaseTransformClass parent_class; } GstCudaVideoConvertScaleClass;

G_DEFINE_TYPE (GstCudaVideoConvertScale, gst_cuda_video_convert_scale, GST_TYPE_BASE_TRANSFORM);

#define GST_TYPE_B200_SCALE_METHOD (gst_b200_scale_method_get_type ())
static GType
gst_b200_scale_method_get_type (void)
{
  static GType t = 0;
  /* nicks and values of GstVideoScaleMethod (gstvideoconvertscale.h:59-71) */
  static const GEnumValue v[] = {
    {B200_SCALE_NEAREST, "Nearest Neighbour", "nearest-neighbour"},
    {B200_SCALE_BILINEAR, "Bilinear (2-tap)", "bilinear"},
    {B200_SCALE_4TAP, "4-tap Sinc", "4-tap"},
    {B200_SCALE_LANCZOS, "Lanczos", "lanczos"},
    {B200_SCALE_BILINEAR2, "Bilinear (multi-tap)", "bilinear2"},
    {B200_SCALE_SINC, "Sinc (multi-tap)", "sinc"},
    {B200_SCALE_HERMITE, "Hermite (multi-tap)", "hermite"},
    {B200_SCALE_SPLINE, "Spline (multi-tap)", "spline"},
    {B200_SCALE_CATROM, "Catmull-Rom (multi-tap)", "catrom"},
    {B200_SCALE_MITCHELL, "Mitchell (multi-tap)", "mitchell"},
    {0, NULL, NULL}
  };
  if (g_once_init_enter (&t))
    g_once_init_leave (&t, g_enum_register_static ("GstB200VideoScaleMethod", v));
  return t;
}

static void
vcs_set_property (GObject * obj, guint id, const GValue * value, GParamSpec * pspec)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) obj;
  GST_OBJECT_LOCK (self);
  switch (id) {
    case PROP_METHOD: self->method = g_value_get_enum (value); break;
    case PROP_ENVELOPE: self->envelope = g_value_get_double (value); break;
    case PROP_SHARPNESS: self->sharpness = g_value_get_double (value); break;
    case PROP_SHARPEN: self->sharpen = g_value_get_double (value); break;
    case PROP_ADD_BORDERS: self->add_borders = g_value_get_boolean (value); break;
    case PROP_DEVICE_ID: self->device_id = g_value_get_int (value); break;
    case PROP_DITHER: self->dither = g_value_get_enum (value); break;
    case PROP_N_THREADS: self->n_threads = g_value_get_uint (value); break;
    case PROP_DITHER_QUANTIZATION: self->dither_quantization = g_value_get_uint (value); break;
    case PROP_CHROMA_RESAMPLER: self->chroma_resampler = g_value_get_enum (value); break;
    case PROP_ALPHA_MODE: self->alpha_mode = g_value_get_enum (value); break;
    case PROP_ALPHA_VALUE: self->alpha_value = g_value_get_double (value); break;
    case PROP_CHROMA_MODE: self->chroma_mode = g_value_get_enum (value); break;
    case PROP_MATRIX_MODE: self->matrix_mode = g_value_get_enum (value); break;
    case PROP_GAMMA_MODE: self->gamma_mode = g_value_get_enum (value); break;
    case PROP_PRIMARIES_MODE: self->primaries_mode = g_value_get_enum (value); break;
    default: G_OBJECT_WARN_INVALID_PROPERTY_ID (obj, id, pspec); break;
  }
  /* like the stock element, the converter is rebuilt lazily on the streaming thread
   * (gstvideoconvertscale.c:1989-2000) */
  self->config_changed = TRUE;
  GST_OBJECT_UNLOCK (self);
}

static void
vcs_get_property (GObject * obj, guint id, GValue * value, GParamSpec * pspec)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) obj;
  GST_OBJECT_LOCK (self);
  switch (id) {
    case PROP_METHOD: g_value_set_enum (value, self->method); break;
    case PROP_ENVELOPE: g_value_set_double (value, self->envelope); break;
    case PROP_SHARPNESS: g_value_set_double (value, self->sharpness); break;
    case PROP_SHARPEN: g_value_set_double (value, self->sharpen); break;
    case PROP_ADD_BORDERS: g_value_set_boolean (value, self->add_borders); break;
    case PROP_DEVICE_ID: g_value_set_int (value, self->device_id); break;
    case PROP_DITHER: g_value_set_enum (value, self->dither); break;
    case PROP_N_THREADS: g_value_set_uint (value, self->n_threads); break;
    case PROP_DITHER_QUANTIZATION: g_value_set_uint (value, self->dither_quantization); break;
    case PROP_CHROMA_RESAMPLER: g_value_set_enum (value, self->chroma_resampler); break;
    case PROP_ALPHA_MODE: g_value_set_enum (value, self->alpha_mode); break;
    case PROP_ALPHA_VALUE: g_value_set_double (value, self->alpha_value); break;
    case PROP_CHROMA_MODE: g_value_set_enum (value, self->chroma_mode); break;
    case PROP_MATRIX_MODE: g_value_set_enum (value, self->matrix_mode); break;
    case PROP_GAMMA_MODE: g_value_set_enum (value, self->gamma_mode); break;
    case PROP_PRIMARIES_MODE: g_value_set_enum (value, self->primaries_mode); break;
    default: G_OBJECT_WARN_INVALID_PROPERTY_ID (obj, id, pspec); break;
  }
  GST_OBJECT_UNLOCK (self);
}

static void
vcs_set_context (GstElement * element, GstContext * context)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) element;
  gst_cuda_handle_set_context (element, context, self->device_id, &self->context);
  GST_ELEMENT_CLASS (gst_cuda_video_convert_scale_parent_class)->set_context (element, context);
}

static gboolean
vcs_start (GstBaseTransform * trans)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) trans;
  if (!gst_cuda_ensure_element_context (GST_ELEMENT (self), self->device_id, &self->context)) {
    GST_ERROR_OBJECT (self, "no CUDA context (libb200dsp has no CPU fallback)");
    return FALSE;
  }
  self->stream = gst_cuda_stream_new (self->context);
  return TRUE;
}

static gboolean
vcs_stop (GstBaseTransform * trans)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) trans;
  if (self->vcs && self->context && gst_cuda_context_push (self->context)) {
    g_clear_pointer (&self->vcs, b200_vcs_destroy);    /* frees device tables: in the context that owns them */
    gst_cuda_context_pop (NULL);
  }
  gst_clear_cuda_stream (&self->stream);
  gst_clear_object (&self->context);
  return TRUE;
}

static gboolean
vcs_query (GstBaseTransform * trans, GstPadDirection direction, GstQuery * query)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) trans;
  if (GST_QUERY_TYPE (query) == GST_QUERY_CONTEXT &&
      gst_cuda_handle_context_query (GST_ELEMENT (self), query, self->context))
    return TRUE;
  return GST_BASE_TRANSFORM_CLASS (gst_cuda_video_convert_scale_parent_class)->query (trans, direction, query);
}

/* 0: 4:2:0, 1: packed RGB, 2: planar 4:2:2 / 4:4:4, 3: packed 4:2:2, 4: planar RGB, -1: not a fixed format name of ours
 * (no name of one class is a substring of a name of another) */
static gint
vcs_format_class (const GstStructure * st)
{
  const gchar *f = gst_structure_get_string (st, "format");
  if (!f)
    return -1;
  if (strstr (YUV420_FORMATS, f))
    return 0;
  if (strstr (RGB_FORMATS, f))
    return 1;
  if (strstr (PLANAR4XX_FORMATS, f))
    return 2;
  if (strstr (PACKED422_FORMATS, f))
    return 3;
  if (strstr (PLANAR_RGB_FORMATS, f))
    return 4;
  return -1;
}

/* caps on the other pad: every format of the other direction, any size in range, colorimetry/chroma-site dropped
 * (gstvideoconvertscale.c:703-748) */
static GstCaps *
vcs_transform_caps (GstBaseTransform * trans, GstPadDirection direction, GstCaps * caps, GstCaps * filter)
{
  GstCaps *tmpl, *res;
  guint i, n;
  (void) trans;
  tmpl = gst_static_pad_template_get_caps (direction == GST_PAD_SINK ? &src_tmpl : &sink_tmpl);
  res = gst_caps_new_empty ();
  n = gst_caps_get_size (caps);
  for (i = 0; i < n; i++) {
    GstStructure *in = gst_caps_get_structure (caps, i);
    GstCaps *one = gst_caps_copy (tmpl);            /* every sink format converts to every src format */
    const GValue *fr = gst_structure_get_value (in, "framerate");
    if (fr)
      gst_caps_set_value (one, "framerate", fr);       /* framerate and interlace-mode pass through */
    gst_caps_append (res, one);
  }
  gst_caps_unref (tmpl);
  if (filter) {
    GstCaps *t = gst_caps_intersect_full (filter, res, GST_CAPS_INTERSECT_FIRST);
    gst_caps_unref (res);
    res = t;
  }
  return res;
}

/* what transfer_colorimetry_from_input does in the stock element (gstvideoconvertscale.c:1335-1427): a YUV output of
 * a YUV input takes the input's colorimetry intact and - the sub-sampling is 4:2:0 on both sides here - its
 * chroma-site; that is what keeps the NV12 <-> I420 chain free of a matrix stage (b200_vcs_create refuses one).
 * Across an RGB <-> YUV change the output keeps the defaults of its own size. */
static void
vcs_transfer_colorimetry (GstCaps * in_caps, GstCaps * out_caps)
{
  GstStructure *in = gst_caps_get_structure (in_caps, 0), *out = gst_caps_get_structure (out_caps, 0);
  const gchar *fi = gst_structure_get_string (in, "format"), *fo = gst_structure_get_string (out, "format");
  const GValue *v;
  if (!fi || !fo)
    return;
  if (!GST_VIDEO_FORMAT_INFO_IS_YUV (gst_video_format_get_info (gst_video_format_from_string (fi))) ||
      !GST_VIDEO_FORMAT_INFO_IS_YUV (gst_video_format_get_info (gst_video_format_from_string (fo))))
    return;
  if (!gst_structure_has_field (out, "colorimetry") && (v = gst_structure_get_value (in, "colorimetry")))
    gst_structure_set_value (out, "colorimetry", v);
  /* the chroma-site travels only across an unchanged sub-sampling (subsampling_unchanged, gstvideoconvertscale.c:1411-1424):
   * a packed 4:2:2 input leaves a 4:2:0 output the default site of its own size */
  if (vcs_format_class (in) == vcs_format_class (out) && !gst_structure_has_field (out, "chroma-site") &&
      (v = gst_structure_get_value (in, "chroma-site")))
    gst_structure_set_value (out, "chroma-site", v);
}

/* fixate_caps (gstvideoconvertscale.c:1431-1960, reduced to what this element negotiates): prefer the input format
 * and size when the peer allows them, carry the colorimetry over, let the default fixation settle the rest */
static GstCaps *
vcs_fixate_caps (GstBaseTransform * trans, GstPadDirection direction, GstCaps * caps, GstCaps * othercaps)
{
  GstStructure *in = gst_caps_get_structure (caps, 0), *out;
  const gchar *fmt = gst_structure_get_string (in, "format");
  gint w = 0, h = 0;
  (void) trans;
  othercaps = gst_caps_truncate (gst_caps_make_writable (othercaps));
  out = gst_caps_get_structure (othercaps, 0);
  if (fmt && gst_structure_has_field (out, "format"))
    gst_structure_fixate_field_string (out, "format", fmt);
  if (gst_structure_get_int (in, "width", &w))
    gst_structure_fixate_field_nearest_int (out, "width", w);
  if (gst_structure_get_int (in, "height", &h))
    gst_structure_fixate_field_nearest_int (out, "height", h);
  othercaps = gst_caps_fixate (othercaps);
  if (direction == GST_PAD_SINK)
    vcs_transfer_colorimetry (caps, othercaps);
  return othercaps;
}

static gboolean
vcs_rebuild (GstCudaVideoConvertScale * self)
{
  b200_video_info in, out;
  b200_vcs_config cfg;
  int st;
  b200_vcs_config_init (&cfg);
  GST_OBJECT_LOCK (self);
  /* dither only acts when quantising (8 -> 8 bit at dither-quantization 1 never does, video-converter.c:2056-2079);
   * n-threads does not change the arithmetic except the reference's chroma pairing at slab boundaries */
  if (self->dither_quantization != 1 || self->chroma_resampler != GST_VIDEO_RESAMPLER_METHOD_LINEAR ||
      self->alpha_mode != GST_VIDEO_ALPHA_MODE_COPY || self->alpha_value != 1.0 ||
      self->chroma_mode != GST_VIDEO_CHROMA_MODE_FULL || self->matrix_mode != GST_VIDEO_MATRIX_MODE_FULL ||
      self->gamma_mode != GST_VIDEO_GAMMA_MODE_NONE || self->primaries_mode != GST_VIDEO_PRIMARIES_MODE_NONE) {
    GST_OBJECT_UNLOCK (self);
    GST_ERROR_OBJECT (self, "only the default of dither-quantization, chroma-resampler, alpha-mode, alpha-value, "
        "chroma-mode, matrix-mode, gamma-mode and primaries-mode is implemented");
    return FALSE;
  }
  cfg.method = self->method;
  cfg.envelope = self->envelope;
  cfg.sharpness = self->sharpness;
  cfg.sharpen = self->sharpen;
  if (self->add_borders) {
    /* gst_video_convert_scale_set_info (gstvideoconvertscale.c:920-952): when the display aspect ratio changes, scale
     * into a centred rectangle that keeps it and let the converter fill the rest with opaque black */
    const GstVideoInfo *ii = &self->in_info, *oi = &self->out_info;
    gint fn, fd, tn, td, n, d, bw = 0, bh = 0;
    if (gst_util_fraction_multiply (ii->width, ii->height, ii->par_n, ii->par_d, &fn, &fd) &&
        gst_util_fraction_multiply (oi->width, oi->height, oi->par_n, oi->par_d, &tn, &td) &&
        (fn != tn || fd != td) && gst_util_fraction_multiply (fn, fd, oi->par_d, oi->par_n, &n, &d)) {
      gint to_h = (gint) gst_util_uint64_scale_int (oi->width, d, n);
      if (to_h <= oi->height)
        bh = oi->height - to_h;
      else
        bw = oi->width - (gint) gst_util_uint64_scale_int (oi->height, n, d);
    }
    cfg.dest_x = bw / 2;
    cfg.dest_y = bh / 2;
    cfg.dest_width = oi->width - bw;
    cfg.dest_height = oi->height - bh;
  }
  self->config_changed = FALSE;
  GST_OBJECT_UNLOCK (self);
  gst_b200_video_info_from_gst (&in, &self->in_info);
  gst_b200_video_info_from_gst (&out, &self->out_info);
  /* every b200 call runs with the element's GstCudaContext current: the library's runtime-API allocations (tap tables,
   * staging slots) must live in the context the frames live in (gstcudacontext.cpp:417 creates a non-primary one) */
  if (!self->context || !gst_cuda_context_push (self->context))
    return FALSE;
  g_clear_pointer (&self->vcs, b200_vcs_destroy);
  st = b200_vcs_create (&in, &out, &cfg, self->device_id, &self->vcs);
  gst_cuda_context_pop (NULL);
  if (st != B200_OK) {
    GST_ERROR_OBJECT (self, "b200_vcs_create: %s", b200_strerror (st));
    return FALSE;                                      /* -> not negotiated */
  }
  return TRUE;
}

static gboolean
vcs_set_caps (GstBaseTransform * trans, GstCaps * incaps, GstCaps * outcaps)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) trans;
  if (!gst_video_info_from_caps (&self->in_info, incaps) || !gst_video_info_from_caps (&self->out_info, outcaps))
    return FALSE;
  if (self->in_info.interlace_mode != self->out_info.interlace_mode)
    return FALSE;                                      /* gstvideoconvertscale.c:958-960 */
  return vcs_rebuild (self);
}

static GstFlowReturn
vcs_transform (GstBaseTransform * trans, GstBuffer * inbuf, GstBuffer * outbuf)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) trans;
  GstVideoFrame in_frame, out_frame;
  GstMemory *in_mem = gst_buffer_peek_memory (inbuf, 0), *out_mem = gst_buffer_peek_memory (outbuf, 0);
  GstCudaStream *in_stream, *out_stream, *use;
  int st;

  if (self->config_changed && !vcs_rebuild (self))
    return GST_FLOW_NOT_NEGOTIATED;
  if (!gst_is_cuda_memory (in_mem) || !gst_is_cuda_memory (out_mem)) {
    /* system-memory peers: plain maps (a GstCudaMemory on one side maps through its own staging) and the library's
     * host entry point: upload, kernel and download pipelined over its device slots */
    const void *src;
    void *dst;
    if (!gst_video_frame_map (&in_frame, &self->in_info, inbuf, GST_MAP_READ))
      return GST_FLOW_ERROR;
    if (!gst_video_frame_map (&out_frame, &self->out_info, outbuf, GST_MAP_WRITE)) {
      gst_video_frame_unmap (&in_frame);
      return GST_FLOW_ERROR;
    }
    src = GST_VIDEO_FRAME_PLANE_DATA (&in_frame, 0);
    dst = GST_VIDEO_FRAME_PLANE_DATA (&out_frame, 0);
    gst_cuda_context_push (self->context);
    st = b200_vcs_convert_host (self->vcs, 1, &src, &dst);
    gst_cuda_context_pop (NULL);
    gst_video_frame_unmap (&out_frame);
    gst_video_frame_unmap (&in_frame);
    GST_B200_FLOW_FROM_STATUS (self, st, "b200_vcs_convert_host");
    return GST_FLOW_OK;
  }

  in_stream = gst_cuda_memory_get_stream (GST_CUDA_MEMORY_CAST (in_mem));
  out_stream = gst_cuda_memory_get_stream (GST_CUDA_MEMORY_CAST (out_mem));
  /* stream choice as gstcudaconvertscale.c:1549-1565: downstream's, else upstream's, else ours */
  use = out_stream ? out_stream : (in_stream ? in_stream : self->stream);
  if (out_stream && in_stream && in_stream != out_stream)
    gst_cuda_memory_sync (GST_CUDA_MEMORY_CAST (in_mem));

  if (!gst_video_frame_map (&in_frame, &self->in_info, inbuf, GST_MAP_READ | GST_MAP_CUDA))
    return GST_FLOW_ERROR;
  if (!gst_video_frame_map (&out_frame, &self->out_info, outbuf, GST_MAP_WRITE | GST_MAP_CUDA)) {
    gst_video_frame_unmap (&in_frame);
    return GST_FLOW_ERROR;
  }
  gst_cuda_context_push (self->context);
  /* plane 0 is the frame base; the library adds the per-plane offsets it was created with */
  st = b200_vcs_convert (self->vcs, GST_VIDEO_FRAME_PLANE_DATA (&in_frame, 0),
      GST_VIDEO_FRAME_PLANE_DATA (&out_frame, 0), gst_cuda_stream_get_handle (use));
  if (st == B200_OK && use != out_stream) {
    /* downstream is not stream aware: finish before the buffer leaves (gstcudaconvertscale.c:1573-1579) */
    GST_MEMORY_FLAG_UNSET (out_mem, GST_CUDA_MEMORY_TRANSFER_NEED_SYNC);
    CuStreamSynchronize (gst_cuda_stream_get_handle (use));
  }
  gst_cuda_context_pop (NULL);
  gst_video_frame_unmap (&out_frame);
  gst_video_frame_unmap (&in_frame);
  GST_B200_FLOW_FROM_STATUS (self, st, "b200_vcs_convert");
  return GST_FLOW_OK;
}

static gboolean
vcs_caps_are_cuda (GstCaps * caps)
{
  GstCapsFeatures *f = caps && gst_caps_get_size (caps) ? gst_caps_get_features (caps, 0) : NULL;
  return f && gst_caps_features_contains (f, GST_CAPS_FEATURE_MEMORY_CUDA_MEMORY);
}

/* propose_allocation (pattern: GstVideoFilter, gst-libs/gst/video/gstvideofilter.c:56-115): offer upstream a pool for
 * our sink caps - a GstCudaBufferPool for CUDA caps, a plain video pool for system memory - and GstVideoMeta, so that
 * strides other than the default reach transform() through the frame map */
static gboolean
vcs_propose_allocation (GstBaseTransform * trans, GstQuery * decide_query, GstQuery * query)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) trans;
  GstCaps *caps;
  GstVideoInfo info;
  GstBufferPool *pool;
  GstStructure *config;
  gboolean need_pool;
  if (decide_query == NULL)                              /* pass-through: let the query travel */
    return GST_BASE_TRANSFORM_CLASS (gst_cuda_video_convert_scale_parent_class)->propose_allocation (trans, decide_query, query);
  gst_query_parse_allocation (query, &caps, &need_pool);
  if (caps == NULL || !gst_video_info_from_caps (&info, caps))
    return FALSE;
  if (need_pool) {
    pool = vcs_caps_are_cuda (caps) && self->context ? gst_cuda_buffer_pool_new (self->context) : gst_video_buffer_pool_new ();
    config = gst_buffer_pool_get_config (pool);
    gst_buffer_pool_config_set_params (config, caps, GST_VIDEO_INFO_SIZE (&info), 0, 0);
    gst_buffer_pool_config_add_option (config, GST_BUFFER_POOL_OPTION_VIDEO_META);
    if (!gst_buffer_pool_set_config (pool, config)) {
      gst_object_unref (pool);
      return FALSE;
    }
    gst_query_add_allocation_pool (query, pool, GST_VIDEO_INFO_SIZE (&info), 0, 0);
    gst_object_unref (pool);
  }
  gst_query_add_allocation_meta (query, GST_VIDEO_META_API_TYPE, NULL);
  return TRUE;
}

static gboolean
vcs_decide_allocation (GstBaseTransform * trans, GstQuery * query)
{
  GstCudaVideoConvertScale *self = (GstCudaVideoConvertScale *) trans;
  GstCaps *caps;
  GstBufferPool *pool = NULL;
  GstStructure *config;
  guint size = GST_VIDEO_INFO_SIZE (&self->out_info), min = 0, max = 0;
  gst_query_parse_allocation (query, &caps, NULL);
  if (!vcs_caps_are_cuda (caps))                        /* system-memory downstream: the base class picks its pool */
    return GST_BASE_TRANSFORM_CLASS (gst_cuda_video_convert_scale_parent_class)->decide_allocation (trans, query);
  if (gst_query_get_n_allocation_pools (query) > 0)
    gst_query_parse_nth_allocation_pool (query, 0, &pool, &size, &min, &max);
  if (pool && !GST_IS_CUDA_BUFFER_POOL (pool))
    gst_clear_object (&pool);
  if (!pool)
    pool = gst_cuda_buffer_pool_new (self->context);
  config = gst_buffer_pool_get_config (pool);
  gst_buffer_pool_config_set_params (config, caps, size, min, max);
  gst_buffer_pool_config_add_option (config, GST_BUFFER_POOL_OPTION_VIDEO_META);
  gst_buffer_pool_set_config (pool, config);
  if (gst_query_get_n_allocation_pools (query) > 0)
    gst_query_set_nth_allocation_pool (query, 0, pool, size, min, max);
  else
    gst_query_add_allocation_pool (query, pool, size, min, max);
  gst_object_unref (pool);
  return TRUE;
}

static void
gst_cuda_video_convert_scale_class_init (GstCudaVideoConvertScaleClass * klass)
{
  GObjectClass *gobject = G_OBJECT_CLASS (klass);
  GstElementClass *element = GST_ELEMENT_CLASS (klass);
  GstBaseTransformClass *trans = GST_BASE_TRANSFORM_CLASS (klass);

  gobject->set_property = vcs_set_property;
  gobject->get_property = vcs_get_property;
  g_object_class_install_property (gobject, PROP_METHOD, g_param_spec_enum ("method", "method", "scaling method",
          GST_TYPE_B200_SCALE_METHOD, B200_SCALE_BILINEAR, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_ENVELOPE, g_param_spec_double ("envelope", "Envelope",
          "Size of filter envelope", 1.0, 5.0, 2.0, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_SHARPNESS, g_param_spec_double ("sharpness", "Sharpness",
          "Sharpness of filter", 0.5, 1.5, 1.0, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_SHARPEN, g_param_spec_double ("sharpen", "Sharpen",
          "Sharpening", 0.0, 1.0, 0.0, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_DITHER, g_param_spec_enum ("dither", "Dither", "Apply dithering while converting",
          gst_video_dither_method_get_type (), GST_VIDEO_DITHER_BAYER, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_N_THREADS, g_param_spec_uint ("n-threads", "Threads",
          "Maximum number of threads to use (accepted; the GPU path has no use for it)", 0, G_MAXUINT, 1,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_DITHER_QUANTIZATION, g_param_spec_uint ("dither-quantization",
          "Dither Quantize", "Quantizer to use", 0, G_MAXUINT, 1, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_CHROMA_RESAMPLER, g_param_spec_enum ("chroma-resampler", "Chroma resampler",
          "Chroma resampler method", gst_video_resampler_method_get_type (), GST_VIDEO_RESAMPLER_METHOD_LINEAR,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_ALPHA_MODE, g_param_spec_enum ("alpha-mode", "Alpha Mode",
          "Alpha Mode to use", gst_video_alpha_mode_get_type (), GST_VIDEO_ALPHA_MODE_COPY,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_ALPHA_VALUE, g_param_spec_double ("alpha-value", "Alpha Value",
          "Alpha Value to use", 0.0, 1.0, 1.0, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_CHROMA_MODE, g_param_spec_enum ("chroma-mode", "Chroma Mode",
          "Chroma Resampling Mode", gst_video_chroma_mode_get_type (), GST_VIDEO_CHROMA_MODE_FULL,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_MATRIX_MODE, g_param_spec_enum ("matrix-mode", "Matrix Mode",
          "Matrix Conversion Mode", gst_video_matrix_mode_get_type (), GST_VIDEO_MATRIX_MODE_FULL,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_GAMMA_MODE, g_param_spec_enum ("gamma-mode", "Gamma Mode",
          "Gamma Conversion Mode", gst_video_gamma_mode_get_type (), GST_VIDEO_GAMMA_MODE_NONE,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_PRIMARIES_MODE, g_param_spec_enum ("primaries-mode", "Primaries Mode",
          "Primaries Conversion Mode", gst_video_primaries_mode_get_type (), GST_VIDEO_PRIMARIES_MODE_NONE,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_ADD_BORDERS, g_param_spec_boolean ("add-borders", "Add Borders",
          "Add black borders if necessary to keep the display aspect ratio", TRUE,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_DEVICE_ID, g_param_spec_int ("cuda-device-id", "Cuda Device ID",
          "Set the GPU device to use for operations (-1 = auto)", -1, G_MAXINT, 0,
          G_PARAM_READWRITE | GST_PARAM_MUTABLE_READY | G_PARAM_STATIC_STRINGS));

  gst_element_class_add_static_pad_template (element, &sink_tmpl);
  gst_element_class_add_static_pad_template (element, &src_tmpl);
  gst_element_class_set_static_metadata (element, "CUDA colourspace converter and scaler",
      "Filter/Converter/Video/Scaler/Colorspace/Hardware",
      "Bit-exact videoconvertscale on sm_90a (libb200dsp)", "b200-gst-dsp");
  element->set_context = vcs_set_context;

  trans->passthrough_on_same_caps = TRUE;
  trans->start = vcs_start;
  trans->stop = vcs_stop;
  trans->query = vcs_query;
  trans->transform_caps = vcs_transform_caps;
  trans->fixate_caps = vcs_fixate_caps;
  trans->set_caps = vcs_set_caps;
  trans->transform = vcs_transform;
  trans->propose_allocation = vcs_propose_allocation;
  trans->decide_allocation = vcs_decide_allocation;
  GST_DEBUG_CATEGORY_INIT (cuda_vcs_debug, "cudavideoconvertscale", 0, "CUDA convert + scale");
}

static void
gst_cuda_video_convert_scale_init (GstCudaVideoConvertScale * self)
{
  self->method = B200_SCALE_BILINEAR;
  self->envelope = 2.0;
  self->sharpness = 1.0;
  self->sharpen = 0.0;
  self->add_borders = TRUE;
  self->dither = GST_VIDEO_DITHER_BAYER;
  self->n_threads = 1;
  self->dither_quantization = 1;
  self->chroma_resampler = GST_VIDEO_RESAMPLER_METHOD_LINEAR;
  self->alpha_mode = GST_VIDEO_ALPHA_MODE_COPY;
  self->alpha_value = 1.0;
  self->chroma_mode = GST_VIDEO_CHROMA_MODE_FULL;
  self->matrix_mode = GST_VIDEO_MATRIX_MODE_FULL;
  self->gamma_mode = GST_VIDEO_GAMMA_MODE_NONE;
  self->primaries_mode = GST_VIDEO_PRIMARIES_MODE_NONE;
  self->device_id = 0;
}
