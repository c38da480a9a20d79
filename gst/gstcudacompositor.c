/* gst/gstcudacompositor.c — `cudacompositor` (element name of the plugin's GstVideoAggregator)
 *
 * Drop-in for `compositor` on CUDA memory: same `background` property (gst-plugins-base/gst/compositor/compositor.c:742)
 * and pad properties xpos / ypos / width / height / sizing-policy / alpha / operator (:190-196); aggregate_frames() hands
 * every pad frame to ONE b200_comp_blend_convert() call where the stock element runs blend_pads() over row slabs
 * (:1739-1887, :1678-1697).  Pads are convert pads (GstVideoAggregatorConvertPad): a pad whose conversion info differs
 * from its caps gets a b200_vcs (method mitchell = the option-less GstVideoConverter) that the library runs inside the
 * blend call.  CUDA plumbing as gst-plugins-bad/sys/nvcodec/gstcudacompositor.cpp.
 *
 * NOT compiled in the development image (no GLib/GStreamer there); see INTEGRATION.md.
 */
#include <gst/video/gstvideoaggregator.h>
#include <gst/cuda/gstcuda.h>

#include "gstb200elements.h"

GST_DEBUG_CATEGORY_STATIC (cuda_comp_debug);
#define GST_CAT_DEFAULT cuda_comp_debug

/* Y444 / Y42B and the little-endian 10 / 12 / 16-bit planar formats blend pads that already have the aggregator's format
 * (blend.c:596-646); convert pads (b200_vcs) exist for the 8-bit 4:2:0 and packed RGB formats.  Sink pads also take every
 * format b200_vcs_create accepts as input; a conversion it declines fails negotiation. */
#define COMP_SINK_FORMATS "{ RGBA, BGRA, ARGB, ABGR, RGBx, BGRx, xRGB, xBGR, I420, YV12, NV12, NV21, YUY2, UYVY, YVYU, Y444, Y42B, " \
    "I420_10LE, I420_12LE, I422_10LE, I422_12LE, Y444_10LE, Y444_12LE, Y444_16LE }"
#define COMP_FORMATS "{ RGBA, BGRA, ARGB, ABGR, I420, YV12, NV12, NV21, Y444, Y42B, I420_10LE, I420_12LE, " \
    "I422_10LE, I422_12LE, Y444_10LE, Y444_12LE, Y444_16LE }"
#define COMP_FIELDS "format = (string) " COMP_FORMATS \
    ", width = (int) [ 1, 32767 ], height = (int) [ 1, 32767 ], framerate = (fraction) [ 0/1, max ]"
/* device memory preferred; system memory (packed RGB) goes through b200_comp_blend_host */
#define COMP_CAPS "video/x-raw(" GST_CAPS_FEATURE_MEMORY_CUDA_MEMORY "), " COMP_FIELDS "; video/x-raw, " COMP_FIELDS
#define COMP_SINK_FIELDS "format = (string) " COMP_SINK_FORMATS \
    ", width = (int) [ 1, 32767 ], height = (int) [ 1, 32767 ], framerate = (fraction) [ 0/1, max ]"
#define COMP_SINK_CAPS "video/x-raw(" GST_CAPS_FEATURE_MEMORY_CUDA_MEMORY "), " COMP_SINK_FIELDS "; video/x-raw, " COMP_SINK_FIELDS

static GstStaticPadTemplate comp_src = GST_STATIC_PAD_TEMPLATE ("src", GST_PAD_SRC, GST_PAD_ALWAYS,
    GST_STATIC_CAPS (COMP_CAPS));
static GstStaticPadTemplate comp_sink = GST_STATIC_PAD_TEMPLATE ("sink_%u", GST_PAD_SINK, GST_PAD_REQUEST,
    GST_STATIC_CAPS (COMP_SINK_CAPS));

/* ------------------------------------------------------------------ pad */
/* one converter, shared by every pad with the same conversion (equal input caps and layout, equal conversion info) so that
 * their frames run as one batch */
typedef struct
{
  b200_vcs *h;
  b200_video_info in, out;
  gint refs;
} CompConv;

static void
conv_release (CompConv ** c)
{
  if (*c && --(*c)->refs == 0) {
    b200_vcs_destroy ((*c)->h);
    g_free (*c);
  }
  *c = NULL;
}

typedef struct
{
  GstVideoAggregatorPad parent;
  gint xpos, ypos;
  gint width, height;            /* pad properties (compositor.c:686-692): the size of the picture in the output, <= 0 unscaled */
  gint sizing_policy;            /* 0 none, 1 keep-aspect-ratio (compositor.c:714) */
  gint x_offset, y_offset;       /* centring offsets of keep-aspect-ratio, from pad_output_size() */
  gdouble alpha;
  gint op;                       /* b200_comp_operator == GstCompositorOperator numbering */
  CompConv *conv;                /* convert pad: the conversion info differs from the pad's caps */
  void *host_conv;               /* system memory: the converted frame (pinned, b200_host_alloc) */
  gsize host_conv_size;
} GstB200CompositorPad;
typedef struct { GstVideoAggregatorPadClass parent_class; } GstB200CompositorPadClass;
G_DEFINE_TYPE (GstB200CompositorPad, gst_b200_compositor_pad, GST_TYPE_VIDEO_AGGREGATOR_PAD);

enum { PAD_PROP_0, PAD_PROP_XPOS, PAD_PROP_YPOS, PAD_PROP_WIDTH, PAD_PROP_HEIGHT, PAD_PROP_ALPHA, PAD_PROP_OPERATOR,
  PAD_PROP_SIZING_POLICY };

static void
pad_set_property (GObject * obj, guint id, const GValue * value, GParamSpec * pspec)
{
  GstB200CompositorPad *pad = (GstB200CompositorPad *) obj;
  switch (id) {
    case PAD_PROP_XPOS: pad->xpos = g_value_get_int (value); break;
    case PAD_PROP_YPOS: pad->ypos = g_value_get_int (value); break;
    case PAD_PROP_WIDTH: pad->width = g_value_get_int (value); break;
    case PAD_PROP_HEIGHT: pad->height = g_value_get_int (value); break;
    case PAD_PROP_SIZING_POLICY: pad->sizing_policy = g_value_get_int (value); break;
    case PAD_PROP_ALPHA: pad->alpha = g_value_get_double (value); break;
    case PAD_PROP_OPERATOR: pad->op = g_value_get_int (value); break;
    default: G_OBJECT_WARN_INVALID_PROPERTY_ID (obj, id, pspec); break;
  }
}

static void
pad_get_property (GObject * obj, guint id, GValue * value, GParamSpec * pspec)
{
  GstB200CompositorPad *pad = (GstB200CompositorPad *) obj;
  switch (id) {
    case PAD_PROP_XPOS: g_value_set_int (value, pad->xpos); break;
    case PAD_PROP_YPOS: g_value_set_int (value, pad->ypos); break;
    case PAD_PROP_WIDTH: g_value_set_int (value, pad->width); break;
    case PAD_PROP_HEIGHT: g_value_set_int (value, pad->height); break;
    case PAD_PROP_SIZING_POLICY: g_value_set_int (value, pad->sizing_policy); break;
    case PAD_PROP_ALPHA: g_value_set_double (value, pad->alpha); break;
    case PAD_PROP_OPERATOR: g_value_set_int (value, pad->op); break;
    default: G_OBJECT_WARN_INVALID_PROPERTY_ID (obj, id, pspec); break;
  }
}

static void
pad_release_conversion (GstB200CompositorPad * pad)
{
  conv_release (&pad->conv);
  g_clear_pointer (&pad->host_conv, b200_host_free);
  pad->host_conv_size = 0;
}

static void
pad_finalize (GObject * obj)
{
  pad_release_conversion ((GstB200CompositorPad *) obj);
  G_OBJECT_CLASS (gst_b200_compositor_pad_parent_class)->finalize (obj);
}

static void
gst_b200_compositor_pad_class_init (GstB200CompositorPadClass * klass)
{
  GObjectClass *gobject = G_OBJECT_CLASS (klass);
  gobject->finalize = pad_finalize;
  gobject->set_property = pad_set_property;
  gobject->get_property = pad_get_property;
  g_object_class_install_property (gobject, PAD_PROP_XPOS, g_param_spec_int ("xpos", "X Position",
          "X Position of the picture", G_MININT, G_MAXINT, 0, G_PARAM_READWRITE | GST_PARAM_CONTROLLABLE));
  g_object_class_install_property (gobject, PAD_PROP_YPOS, g_param_spec_int ("ypos", "Y Position",
          "Y Position of the picture", G_MININT, G_MAXINT, 0, G_PARAM_READWRITE | GST_PARAM_CONTROLLABLE));
  g_object_class_install_property (gobject, PAD_PROP_WIDTH, g_param_spec_int ("width", "Width",
          "Width of the picture", G_MININT, G_MAXINT, 0, G_PARAM_READWRITE | GST_PARAM_CONTROLLABLE));
  g_object_class_install_property (gobject, PAD_PROP_HEIGHT, g_param_spec_int ("height", "Height",
          "Height of the picture", G_MININT, G_MAXINT, 0, G_PARAM_READWRITE | GST_PARAM_CONTROLLABLE));
  g_object_class_install_property (gobject, PAD_PROP_SIZING_POLICY, g_param_spec_int ("sizing-policy", "Sizing policy",
          "0 none, 1 keep-aspect-ratio (GstCompositorSizingPolicy)", 0, 1, 0, G_PARAM_READWRITE | GST_PARAM_CONTROLLABLE));
  g_object_class_install_property (gobject, PAD_PROP_ALPHA, g_param_spec_double ("alpha", "Alpha",
          "Alpha of the picture", 0.0, 1.0, 1.0, G_PARAM_READWRITE | GST_PARAM_CONTROLLABLE));
  g_object_class_install_property (gobject, PAD_PROP_OPERATOR, g_param_spec_int ("operator", "Operator",
          "0 source, 1 over, 2 add (GstCompositorOperator)", 0, 2, 1, G_PARAM_READWRITE | GST_PARAM_CONTROLLABLE));
}

static void
gst_b200_compositor_pad_init (GstB200CompositorPad * pad)
{
  pad->alpha = 1.0;
  pad->op = B200_COMP_OP_OVER;
}

/* _mixer_pad_get_output_size (compositor.c:289-417) for pixel aspect ratio 1/1: the size the pad's picture takes in the
 * output and the offsets that centre it under sizing-policy=keep-aspect-ratio (gst_video_center_rect,
 * gstvideosink.c:122-164).  The pad's converter (b200_vcs, method mitchell = the option-less GstVideoConverter of a
 * GstVideoAggregatorConvertPad) scales to this size; blending happens at xpos + x_offset, ypos + y_offset. */
static void
pad_output_size (GstB200CompositorPad * pad, gboolean zero_size_is_unscaled, gint * width, gint * height)
{
  const GstVideoInfo *info = &GST_VIDEO_AGGREGATOR_PAD (pad)->info;
  gint sw = GST_VIDEO_INFO_WIDTH (info), sh = GST_VIDEO_INFO_HEIGHT (info);
  gint pw = (zero_size_is_unscaled ? pad->width <= 0 : pad->width < 0) ? sw : pad->width;
  gint ph = (zero_size_is_unscaled ? pad->height <= 0 : pad->height < 0) ? sh : pad->height;
  gint fn, fd, tn, td;
  pad->x_offset = pad->y_offset = 0;
  *width = *height = 0;
  if (pw == 0 || ph == 0)
    return;
  if (pad->sizing_policy == 1 && gst_util_fraction_multiply (sw, sh, 1, 1, &fn, &fd) &&
      gst_util_fraction_multiply (pw, ph, 1, 1, &tn, &td) && (fn != tn || fd != td)) {
    gint rh = (gint) gst_util_uint64_scale_int (pw, fd, fn);
    gdouble src_ratio, dst_ratio;
    if (rh == 0)
      return;
    src_ratio = (gdouble) pw / rh;
    dst_ratio = (gdouble) pw / ph;
    if (src_ratio > dst_ratio) {
      gint h = (gint) (pw / src_ratio);
      pad->y_offset = (ph - h) / 2;
      ph = h;
    } else if (src_ratio < dst_ratio) {
      gint w = (gint) (ph * src_ratio);
      pad->x_offset = (pw - w) / 2;
      pw = w;
    }
  }
  *width = pw;
  *height = ph;
}

/* ------------------------------------------------------------------ element */
typedef struct
{
  GstVideoAggregator parent;
  gint background, device_id;
  gboolean zero_size_is_unscaled, ignore_inactive_pads;      /* compositor.c:2117, :2162; defaults TRUE / FALSE */
  guint max_threads;             /* accepted; the single-pass GPU blend has no use for it */
  GstCudaContext *context;
  GstCudaStream *stream;
  b200_comp *comp;
  gint comp_w, comp_h, comp_fmt;
} GstB200CudaCompositor;
typedef struct { GstVideoAggregatorClass parent_class; } GstB200CudaCompositorClass;
G_DEFINE_TYPE (GstB200CudaCompositor, gst_b200_cuda_compositor, GST_TYPE_VIDEO_AGGREGATOR);

enum { PROP_0, PROP_BACKGROUND, PROP_DEVICE_ID, PROP_ZERO_SIZE_IS_UNSCALED, PROP_MAX_THREADS, PROP_IGNORE_INACTIVE_PADS };

static void
comp_set_property (GObject * obj, guint id, const GValue * value, GParamSpec * pspec)
{
  GstB200CudaCompositor *self = (GstB200CudaCompositor *) obj;
  switch (id) {
    case PROP_BACKGROUND: self->background = g_value_get_int (value); break;
    case PROP_DEVICE_ID: self->device_id = g_value_get_int (value); break;
    case PROP_ZERO_SIZE_IS_UNSCALED: self->zero_size_is_unscaled = g_value_get_boolean (value); break;
    case PROP_MAX_THREADS: self->max_threads = g_value_get_uint (value); break;
    case PROP_IGNORE_INACTIVE_PADS: self->ignore_inactive_pads = g_value_get_boolean (value); break;
    default: G_OBJECT_WARN_INVALID_PROPERTY_ID (obj, id, pspec); break;
  }
}

static void
comp_get_property (GObject * obj, guint id, GValue * value, GParamSpec * pspec)
{
  GstB200CudaCompositor *self = (GstB200CudaCompositor *) obj;
  switch (id) {
    case PROP_BACKGROUND: g_value_set_int (value, self->background); break;
    case PROP_DEVICE_ID: g_value_set_int (value, self->device_id); break;
    case PROP_ZERO_SIZE_IS_UNSCALED: g_value_set_boolean (value, self->zero_size_is_unscaled); break;
    case PROP_MAX_THREADS: g_value_set_uint (value, self->max_threads); break;
    case PROP_IGNORE_INACTIVE_PADS: g_value_set_boolean (value, self->ignore_inactive_pads); break;
    default: G_OBJECT_WARN_INVALID_PROPERTY_ID (obj, id, pspec); break;
  }
}

static gboolean
comp_start (GstAggregator * agg)
{
  GstB200CudaCompositor *self = (GstB200CudaCompositor *) agg;
  if (!gst_cuda_ensure_element_context (GST_ELEMENT (self), self->device_id, &self->context))
    return FALSE;
  self->stream = gst_cuda_stream_new (self->context);
  return TRUE;
}

static gboolean
comp_stop (GstAggregator * agg)
{
  GstB200CudaCompositor *self = (GstB200CudaCompositor *) agg;
  GList *l;
  GST_OBJECT_LOCK (agg);
  for (l = GST_ELEMENT (agg)->sinkpads; l; l = l->next)
    pad_release_conversion (l->data);
  GST_OBJECT_UNLOCK (agg);
  g_clear_pointer (&self->comp, b200_comp_destroy);
  gst_clear_cuda_stream (&self->stream);
  gst_clear_object (&self->context);
  return GST_AGGREGATOR_CLASS (gst_b200_cuda_compositor_parent_class)->stop (agg);
}

/* gst_video_aggregator_convert_pad_create_conversion_info + gst_compositor_pad_create_conversion_info
 * (gstvideoaggregator.c:580-640, compositor.c:603-662): the aggregator's format, colorimetry and chroma site at the pad's
 * output size.  FALSE when that is what the pad's caps already are: no conversion. */
static gboolean
pad_conversion_info (const b200_video_info * in, const GstVideoInfo * oinfo, gint w, gint h, b200_video_info * out)
{
  if (b200_video_info_set_format (out, GST_VIDEO_INFO_FORMAT (oinfo), w, h) != B200_OK)
    return TRUE;                 /* an output the converter cannot produce: b200_vcs_create declines it */
  out->color_matrix = oinfo->colorimetry.matrix;
  out->color_range = oinfo->colorimetry.range;
  out->chroma_site = oinfo->chroma_site;
  return !(in->format == out->format && in->width == w && in->height == h && in->color_matrix == out->color_matrix &&
      in->color_range == out->color_range && in->chroma_site == out->chroma_site);
}

/* The pad's converter for in -> out: kept while both stay the same, else released (caps or size properties changed) and
 * taken from another pad with the same conversion, or created - method mitchell, no destination rectangle.  The caller
 * holds the object lock and has the CUDA context pushed. */
static gint
pad_ensure_conv (GstB200CudaCompositor * self, GstB200CompositorPad * cpad, const b200_video_info * in,
    const b200_video_info * out)
{
  b200_vcs_config cfg;
  CompConv *c;
  GList *l;
  gint st;
  if (cpad->conv && !memcmp (&cpad->conv->in, in, sizeof (*in)) && !memcmp (&cpad->conv->out, out, sizeof (*out)))
    return B200_OK;
  pad_release_conversion (cpad);
  for (l = GST_ELEMENT (self)->sinkpads; l; l = l->next) {
    GstB200CompositorPad *other = l->data;
    if (other != cpad && other->conv && !memcmp (&other->conv->in, in, sizeof (*in)) &&
        !memcmp (&other->conv->out, out, sizeof (*out))) {
      cpad->conv = other->conv;
      cpad->conv->refs++;
      return B200_OK;
    }
  }
  b200_vcs_config_init (&cfg);
  cfg.method = B200_SCALE_MITCHELL;
  c = g_new0 (CompConv, 1);
  c->in = *in;
  c->out = *out;
  c->refs = 1;
  st = b200_vcs_create (in, out, &cfg, self->device_id, &c->h);
  if (st != B200_OK) {
    g_free (c);
    return st;
  }
  cpad->conv = c;
  return B200_OK;
}

static GstFlowReturn
comp_aggregate_frames (GstVideoAggregator * vagg, GstBuffer * outbuf)
{
  GstB200CudaCompositor *self = (GstB200CudaCompositor *) vagg;
  GstVideoFrame out_frame;
  b200_comp_pad_convert pads[B200_COMP_MAX_PADS];
  GstB200CompositorPad *cpads[B200_COMP_MAX_PADS];
  b200_video_info di;
  gint n = 0, i, st = B200_OK;
  GList *l;
  const GstVideoInfo *oinfo = &vagg->info;

  if (!self->comp || self->comp_w != GST_VIDEO_INFO_WIDTH (oinfo) || self->comp_h != GST_VIDEO_INFO_HEIGHT (oinfo)
      || self->comp_fmt != (gint) GST_VIDEO_INFO_FORMAT (oinfo)) {
    g_clear_pointer (&self->comp, b200_comp_destroy);
    st = b200_comp_create (GST_VIDEO_INFO_FORMAT (oinfo), GST_VIDEO_INFO_WIDTH (oinfo),
        GST_VIDEO_INFO_HEIGHT (oinfo), self->device_id, &self->comp);
    GST_B200_FLOW_FROM_STATUS (self, st, "b200_comp_create");
    self->comp_w = GST_VIDEO_INFO_WIDTH (oinfo);
    self->comp_h = GST_VIDEO_INFO_HEIGHT (oinfo);
    self->comp_fmt = GST_VIDEO_INFO_FORMAT (oinfo);
  }
  const gboolean on_device = gst_is_cuda_memory (gst_buffer_peek_memory (outbuf, 0));
  if (!gst_video_frame_map (&out_frame, (GstVideoInfo *) oinfo, outbuf, on_device ? (GST_MAP_WRITE | GST_MAP_CUDA) : GST_MAP_WRITE))
    return GST_FLOW_ERROR;
  gst_b200_video_info_from_gst (&di, &out_frame.info);

  /* sink pads in z-order (the aggregator keeps element->sinkpads sorted by zorder); compositor.c:1775-1832 builds the
   * same list.  Each pad's conversion info decides whether it converts; its converter is created or shared here. */
  gst_cuda_context_push (self->context);
  GST_OBJECT_LOCK (vagg);
  for (l = GST_ELEMENT (vagg)->sinkpads; l && n < B200_COMP_MAX_PADS; l = l->next) {
    GstB200CompositorPad *cpad = l->data;
    GstVideoFrame *f = gst_video_aggregator_pad_get_prepared_frame (GST_VIDEO_AGGREGATOR_PAD (cpad));
    b200_video_info conv_info;
    gint pw, ph;
    if (!f)
      continue;
    pad_output_size (cpad, self->zero_size_is_unscaled, &pw, &ph);
    if (pw == 0 || ph == 0)
      continue;                  /* compositor.c:547-550: nothing to draw */
    b200_comp_pad_convert *p = &pads[n];
    memset (p, 0, sizeof (*p));
    p->data = GST_VIDEO_FRAME_PLANE_DATA (f, 0);
    gst_b200_video_info_from_gst (&p->info, &f->info);
    if (pad_conversion_info (&p->info, oinfo, pw, ph, &conv_info)) {
      if ((st = pad_ensure_conv (self, cpad, &p->info, &conv_info)) != B200_OK)
        break;
      p->conv = cpad->conv->h;
    } else {
      pad_release_conversion (cpad);
    }
    p->xpos = cpad->xpos + cpad->x_offset;      /* compositor.c:1692-1693 */
    p->ypos = cpad->ypos + cpad->y_offset;
    p->alpha = cpad->alpha;
    p->op = cpad->op;
    cpads[n++] = cpad;
  }
  GST_OBJECT_UNLOCK (vagg);
  if (st != B200_OK) {
    /* the converter declines this pad's conversion (e.g. a YUV -> YUV colour matrix change): not negotiated rather than
     * blended wrong */
    gst_cuda_context_pop (NULL);
    gst_video_frame_unmap (&out_frame);
    GST_ELEMENT_ERROR (self, CORE, NEGOTIATION, ("pad conversion not supported: %s", b200_strerror (st)), (NULL));
    return GST_FLOW_NOT_NEGOTIATED;
  }

  if (!on_device) {
    /* system-memory peers: converted pads go through b200_vcs_convert_host into a pinned pad-owned frame, then every
     * pad frame and the output are staged by the library's own device ring - upload, one blend pass, download */
    const gboolean yuv = GST_VIDEO_INFO_IS_YUV (oinfo);
    b200_comp_pad rpads[B200_COMP_MAX_PADS];
    b200_comp_pad_yuv ypads[B200_COMP_MAX_PADS];
    for (i = 0; i < n && st == B200_OK; i++) {
      const void *data = pads[i].data;
      const b200_video_info *fi = &pads[i].info;
      if (pads[i].conv) {
        const gsize size = b200_video_info_size (&cpads[i]->conv->out);
        if (cpads[i]->host_conv_size < size) {
          g_clear_pointer (&cpads[i]->host_conv, b200_host_free);
          cpads[i]->host_conv_size = 0;
          if ((st = b200_host_alloc (size, &cpads[i]->host_conv)) != B200_OK)
            break;
          cpads[i]->host_conv_size = size;
        }
        if ((st = b200_vcs_convert_host (pads[i].conv, 1, &pads[i].data, &cpads[i]->host_conv)) != B200_OK)
          break;
        data = cpads[i]->host_conv;
        fi = &cpads[i]->conv->out;
      }
      if (yuv) {
        ypads[i].data = data;
        ypads[i].info = *fi;
        ypads[i].xpos = pads[i].xpos; ypads[i].ypos = pads[i].ypos;
        ypads[i].alpha = pads[i].alpha; ypads[i].op = pads[i].op; ypads[i].reserved = 0;
      } else {
        rpads[i].data = (const guint8 *) data + fi->offset[0];
        rpads[i].width = fi->width;
        rpads[i].height = fi->height;
        rpads[i].stride = fi->stride[0];
        rpads[i].xpos = pads[i].xpos; rpads[i].ypos = pads[i].ypos;
        rpads[i].alpha = pads[i].alpha; rpads[i].op = pads[i].op; rpads[i].reserved = 0;
      }
    }
    if (st == B200_OK)
      st = yuv ? b200_comp_blend_yuv_host (self->comp, GST_VIDEO_FRAME_PLANE_DATA (&out_frame, 0), &di, self->background, ypads, n)
          : b200_comp_blend_host (self->comp, GST_VIDEO_FRAME_PLANE_DATA (&out_frame, 0),
          GST_VIDEO_FRAME_PLANE_STRIDE (&out_frame, 0), self->background, rpads, n);
    gst_cuda_context_pop (NULL);
    gst_video_frame_unmap (&out_frame);
    GST_B200_FLOW_FROM_STATUS (self, st, "b200_comp_blend_host");
    return GST_FLOW_OK;
  }
  /* device memory: conversions and the blend in one call (plane layouts travel as b200_video_info, offsets relative to
   * plane 0) */
  st = b200_comp_blend_convert (self->comp, GST_VIDEO_FRAME_PLANE_DATA (&out_frame, 0), &di, self->background, pads, n,
      gst_cuda_stream_get_handle (self->stream));
  if (st == B200_OK)
    CuStreamSynchronize (gst_cuda_stream_get_handle (self->stream));
  gst_cuda_context_pop (NULL);
  gst_video_frame_unmap (&out_frame);
  GST_B200_FLOW_FROM_STATUS (self, st, "b200_comp_blend_convert");
  return GST_FLOW_OK;
}

static void
gst_b200_cuda_compositor_class_init (GstB200CudaCompositorClass * klass)
{
  GObjectClass *gobject = G_OBJECT_CLASS (klass);
  GstElementClass *element = GST_ELEMENT_CLASS (klass);
  GstAggregatorClass *agg = GST_AGGREGATOR_CLASS (klass);
  GstVideoAggregatorClass *vagg = GST_VIDEO_AGGREGATOR_CLASS (klass);

  gobject->set_property = comp_set_property;
  gobject->get_property = comp_get_property;
  g_object_class_install_property (gobject, PROP_BACKGROUND, g_param_spec_int ("background", "Background",
          "0 checker, 1 black, 2 white, 3 transparent (GstCompositorBackground)", 0, 3, 0,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_ZERO_SIZE_IS_UNSCALED, g_param_spec_boolean ("zero-size-is-unscaled",
          "Zero size is unscaled", "If TRUE, then input video is unscaled in that dimension if width or height is 0",
          TRUE, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_MAX_THREADS, g_param_spec_uint ("max-threads", "Max Threads",
          "Maximum number of blending/rendering worker threads (accepted; the GPU blend is one pass)", 0, G_MAXINT, 0,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_IGNORE_INACTIVE_PADS, g_param_spec_boolean ("ignore-inactive-pads",
          "Ignore inactive pads", "Avoid timing out waiting for inactive pads", FALSE,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_DEVICE_ID, g_param_spec_int ("cuda-device-id", "Cuda Device ID",
          "GPU device to use", -1, G_MAXINT, 0, G_PARAM_READWRITE | GST_PARAM_MUTABLE_READY | G_PARAM_STATIC_STRINGS));
  gst_element_class_add_static_pad_template_with_gtype (element, &comp_src, GST_TYPE_AGGREGATOR_PAD);
  gst_element_class_add_static_pad_template_with_gtype (element, &comp_sink, gst_b200_compositor_pad_get_type ());
  gst_element_class_set_static_metadata (element, "CUDA compositor", "Filter/Editor/Video/Compositor/Hardware",
      "Bit-exact compositor alpha blend in one pass on sm_90a (libb200dsp)", "b200-gst-dsp");
  agg->start = comp_start;
  agg->stop = comp_stop;
  vagg->aggregate_frames = comp_aggregate_frames;
  GST_DEBUG_CATEGORY_INIT (cuda_comp_debug, "cudacompositor", 0, "CUDA compositor");
}

static void
gst_b200_cuda_compositor_init (GstB200CudaCompositor * self)
{
  self->background = B200_COMP_BG_CHECKER;
  self->device_id = 0;
  self->zero_size_is_unscaled = TRUE;
}
