/* gst/gstcudaaudioresample.c — `cudaaudioresample`
 *
 * Drop-in for `audioresample` for F32 interleaved audio: same `quality` property
 * (gst-plugins-base/gst/audioresample/gstaudioresample.c:68, :144-228), same framing rules —
 * output length from the resampler before processing (:763-769), zero-length outputs dropped
 * (:879-882), reset on flush/discont (:462, :907-915), drain with silence on EOS (:590-662),
 * timestamps from running sample counters (:846-866).  Audio buffers are system memory: the FIR runs on the GPU
 * through b200_ars_process_host_submit / _wait, i.e. the LIBRARY owns the device staging ring (sized in the caps'
 * bytes per frame, allocated on the element's device under its own device guard) and the three side streams; the
 * element holds no CUDA state of its own.
 *
 * NOT compiled in the development image (no GLib/GStreamer there); see INTEGRATION.md.
 */
#include <gst/base/gstbasetransform.h>
#include <gst/audio/audio.h>

#include "gstb200elements.h"

GST_DEBUG_CATEGORY_STATIC (cuda_ars_debug);
#define GST_CAT_DEFAULT cuda_ars_debug

/* every sample format, as the stock element (gstaudioresample.c:84-85); interleaved only */
#define ARS_CAPS "audio/x-raw, format = (string) " GST_AUDIO_FORMATS_ALL ", layout = (string) interleaved, " \
    "rate = (int) [ 1, MAX ], channels = (int) [ 1, MAX ]"
static GstStaticPadTemplate ars_sink = GST_STATIC_PAD_TEMPLATE ("sink", GST_PAD_SINK, GST_PAD_ALWAYS, GST_STATIC_CAPS (ARS_CAPS));
static GstStaticPadTemplate ars_src = GST_STATIC_PAD_TEMPLATE ("src", GST_PAD_SRC, GST_PAD_ALWAYS, GST_STATIC_CAPS (ARS_CAPS));

enum { PROP_0, PROP_QUALITY, PROP_DEVICE_ID,
  /* the stock element's remaining properties (gstaudioresample.c:160-186), stock defaults: kaiser and blackman-nuttall,
   * every filter mode, cubic table interpolation or none are implemented; the rest fails set_caps */
  PROP_RESAMPLE_METHOD, PROP_SINC_FILTER_MODE, PROP_SINC_FILTER_AUTO_THRESHOLD, PROP_SINC_FILTER_INTERPOLATION
};

typedef struct
{
  GstBaseTransform parent;
  gint quality, device_id;
  gint method, sinc_filter_mode, sinc_filter_interpolation;
  guint sinc_filter_auto_threshold;
  GstAudioInfo in, out;
  b200_ars *ars;
  /* running position (gstaudioresample.c:846-866) */
  GstClockTime t0;
  guint64 in_offset0, out_offset0, samples_in, samples_out;
  gboolean need_discont;
} GstCudaAudioResample;
typedef struct { GstBaseTransformClass parent_class; } GstCudaAudioResampleClass;
G_DEFINE_TYPE (GstCudaAudioResample, gst_cuda_audio_resample, GST_TYPE_BASE_TRANSFORM);

static void
ars_reset_position (GstCudaAudioResample * self)
{
  self->t0 = GST_CLOCK_TIME_NONE;
  self->samples_in = self->samples_out = 0;
  self->need_discont = TRUE;
  if (self->ars)
    b200_ars_reset (self->ars);
}

static gboolean
ars_set_caps (GstBaseTransform * trans, GstCaps * incaps, GstCaps * outcaps)
{
  GstCudaAudioResample *self = (GstCudaAudioResample *) trans;
  b200_ars_config cfg = { 0, };
  GstAudioInfo in, out;
  if (!gst_audio_info_from_caps (&in, incaps) || !gst_audio_info_from_caps (&out, outcaps))
    return FALSE;
  /* gst_audio_resample_update_state (gstaudioresample.c:398-437): same sample format and channel count on a live
   * resampler is a RATE CHANGE - the converter is updated, history and phase survive (b200_ars_update); anything else
   * builds a new resampler */
  if (self->ars && GST_AUDIO_INFO_FORMAT (&in) == GST_AUDIO_INFO_FORMAT (&self->in) &&
      GST_AUDIO_INFO_CHANNELS (&in) == GST_AUDIO_INFO_CHANNELS (&self->in) &&
      GST_AUDIO_INFO_RATE (&in) != GST_AUDIO_INFO_RATE (&out)) {
    if (b200_ars_update (self->ars, GST_AUDIO_INFO_RATE (&in), GST_AUDIO_INFO_RATE (&out)) != B200_OK)
      return FALSE;
    self->in = in;
    self->out = out;
    return TRUE;
  }
  self->in = in;
  self->out = out;
  g_clear_pointer (&self->ars, b200_ars_destroy);
  /* b200_ars_config carries the reference's enum values + 1 (0 = element default) */
  cfg.resample_method = self->method + 1;
  cfg.sinc_filter_mode = self->sinc_filter_mode + 1;
  cfg.sinc_filter_interpolation = self->sinc_filter_interpolation + 1;
  cfg.in_rate = GST_AUDIO_INFO_RATE (&self->in);
  cfg.out_rate = GST_AUDIO_INFO_RATE (&self->out);
  cfg.channels = GST_AUDIO_INFO_CHANNELS (&self->in);
  cfg.quality = self->quality;
  cfg.format = GST_AUDIO_INFO_FORMAT (&self->in);       /* B200_AUDIO_FORMAT_* are GstAudioFormat values */
  /* equal rates: pass-through, no resampler behind the element (gst_audio_resample_set_caps does the same with
   * gst_base_transform_set_passthrough) */
  if (cfg.in_rate == cfg.out_rate) {
    gst_base_transform_set_passthrough (trans, TRUE);
    ars_reset_position (self);
    return TRUE;
  }
  if (b200_ars_create (&cfg, self->device_id, &self->ars) != B200_OK)
    return FALSE;
  gst_base_transform_set_passthrough (trans, FALSE);
  ars_reset_position (self);
  return TRUE;
}

static gboolean
ars_get_unit_size (GstBaseTransform * trans, GstCaps * caps, gsize * size)
{
  GstAudioInfo info;
  if (!gst_audio_info_from_caps (&info, caps))
    return FALSE;
  *size = GST_AUDIO_INFO_BPF (&info);
  return TRUE;
}

static gboolean
ars_transform_size (GstBaseTransform * trans, GstPadDirection direction, GstCaps * caps, gsize size,
    GstCaps * othercaps, gsize * othersize)
{
  GstCudaAudioResample *self = (GstCudaAudioResample *) trans;
  const gsize bpf = GST_AUDIO_INFO_BPF (&self->in);
  gsize frames = size / bpf;
  if (gst_base_transform_is_passthrough (trans)) {
    *othersize = size;
    return TRUE;
  }
  if (!self->ars)
    return FALSE;
  frames = direction == GST_PAD_SINK ? b200_ars_get_out_frames (self->ars, frames)
      : b200_ars_get_in_frames (self->ars, frames);
  *othersize = frames * bpf;
  return TRUE;
}

static GstFlowReturn
ars_transform (GstBaseTransform * trans, GstBuffer * inbuf, GstBuffer * outbuf)
{
  GstCudaAudioResample *self = (GstCudaAudioResample *) trans;
  const gsize bpf = GST_AUDIO_INFO_BPF (&self->in);
  GstMapInfo imap, omap;
  gsize in_frames, out_frames, got = 0;
  int st;

  if (GST_BUFFER_IS_DISCONT (inbuf))
    ars_reset_position (self);                         /* gstaudioresample.c:907-915 */
  if (!GST_CLOCK_TIME_IS_VALID (self->t0)) {
    self->t0 = GST_BUFFER_PTS (inbuf);
    self->in_offset0 = GST_BUFFER_OFFSET (inbuf);
    self->out_offset0 = gst_util_uint64_scale_int_round (self->in_offset0, GST_AUDIO_INFO_RATE (&self->out),
        GST_AUDIO_INFO_RATE (&self->in));
  }
  if (!gst_buffer_map (inbuf, &imap, GST_MAP_READ))
    return GST_FLOW_ERROR;
  in_frames = imap.size / bpf;
  out_frames = b200_ars_get_out_frames (self->ars, in_frames);
  if (!gst_buffer_map (outbuf, &omap, GST_MAP_WRITE)) {
    gst_buffer_unmap (inbuf, &imap);
    return GST_FLOW_ERROR;
  }
  /* upload -> FIR -> download on the library's streams; GstBaseTransform hands the output on when we return, so this
   * buffer has to be complete: one wait per buffer, no device-wide synchronisation */
  st = b200_ars_process_host_submit (self->ars, GST_BUFFER_FLAG_IS_SET (inbuf, GST_BUFFER_FLAG_GAP) ? NULL : imap.data,
      in_frames, omap.data, MIN (out_frames, omap.size / bpf), &got);
  if (st == B200_OK)
    st = b200_ars_process_host_wait (self->ars, 0);
  gst_buffer_unmap (outbuf, &omap);
  gst_buffer_unmap (inbuf, &imap);
  GST_B200_FLOW_FROM_STATUS (self, st, "b200_ars_process_host");

  gst_buffer_set_size (outbuf, got * bpf);             /* :763-769 */
  GST_BUFFER_PTS (outbuf) = self->t0 + gst_util_uint64_scale_int_round (self->samples_out, GST_SECOND,
      GST_AUDIO_INFO_RATE (&self->out));
  GST_BUFFER_OFFSET (outbuf) = self->out_offset0 + self->samples_out;
  self->samples_in += in_frames;
  self->samples_out += got;
  GST_BUFFER_OFFSET_END (outbuf) = self->out_offset0 + self->samples_out;
  GST_BUFFER_DURATION (outbuf) = self->t0 + gst_util_uint64_scale_int_round (self->samples_out, GST_SECOND,
      GST_AUDIO_INFO_RATE (&self->out)) - GST_BUFFER_PTS (outbuf);
  if (self->need_discont) {
    GST_BUFFER_FLAG_SET (outbuf, GST_BUFFER_FLAG_DISCONT);
    self->need_discont = FALSE;
  }
  return got ? GST_FLOW_OK : GST_BASE_TRANSFORM_FLOW_DROPPED;     /* :879-882 */
}

/* drain: feed get_max_latency() frames of silence and push what comes out (gstaudioresample.c:590-662) */
static void
ars_push_drain (GstCudaAudioResample * self)
{
  GstBaseTransform *trans = GST_BASE_TRANSFORM (self);
  const gsize bpf = GST_AUDIO_INFO_BPF (&self->in);
  gsize in_frames, out_frames, got = 0;
  GstBuffer *outbuf;
  GstMapInfo omap;
  if (!self->ars || gst_base_transform_is_passthrough (trans))
    return;
  in_frames = b200_ars_get_max_latency (self->ars);
  out_frames = b200_ars_get_out_frames (self->ars, in_frames);
  if (out_frames == 0)
    return;
  outbuf = gst_buffer_new_and_alloc (out_frames * bpf);
  if (!gst_buffer_map (outbuf, &omap, GST_MAP_WRITE)) {
    gst_buffer_unref (outbuf);
    return;
  }
  if (b200_ars_process_host (self->ars, NULL, in_frames, omap.data, out_frames, &got) != B200_OK)
    got = 0;
  gst_buffer_unmap (outbuf, &omap);
  if (!got) {
    gst_buffer_unref (outbuf);
    return;
  }
  gst_buffer_set_size (outbuf, got * bpf);
  GST_BUFFER_PTS (outbuf) = self->t0 + gst_util_uint64_scale_int_round (self->samples_out, GST_SECOND,
      GST_AUDIO_INFO_RATE (&self->out));
  self->samples_out += got;
  gst_pad_push (GST_BASE_TRANSFORM_SRC_PAD (trans), outbuf);
}

static gboolean
ars_sink_event (GstBaseTransform * trans, GstEvent * event)
{
  GstCudaAudioResample *self = (GstCudaAudioResample *) trans;
  switch (GST_EVENT_TYPE (event)) {
    case GST_EVENT_FLUSH_STOP: ars_reset_position (self); break;
    case GST_EVENT_SEGMENT: ars_push_drain (self); ars_reset_position (self); break;
    case GST_EVENT_EOS: ars_push_drain (self); break;
    default: break;
  }
  return GST_BASE_TRANSFORM_CLASS (gst_cuda_audio_resample_parent_class)->sink_event (trans, event);
}

static gboolean
ars_start (GstBaseTransform * trans)
{
  GstCudaAudioResample *self = (GstCudaAudioResample *) trans;
  (void) self;
  return b200_device_count () > 0;                      /* no CPU fallback: refuse to start without a device */
}

static gboolean
ars_stop (GstBaseTransform * trans)
{
  GstCudaAudioResample *self = (GstCudaAudioResample *) trans;
  g_clear_pointer (&self->ars, b200_ars_destroy);     /* frees the staging ring and the streams with it */
  return TRUE;
}

static GstCaps *
ars_transform_caps (GstBaseTransform * trans, GstPadDirection direction, GstCaps * caps, GstCaps * filter)
{
  /* everything but the rate passes through (gstaudioresample.c:296-330) */
  GstCaps *res = gst_caps_copy (caps);
  guint i;
  for (i = 0; i < gst_caps_get_size (res); i++)
    gst_structure_set (gst_caps_get_structure (res, i), "rate", GST_TYPE_INT_RANGE, 1, G_MAXINT, NULL);
  if (filter) {
    GstCaps *t = gst_caps_intersect_full (filter, res, GST_CAPS_INTERSECT_FIRST);
    gst_caps_unref (res);
    res = t;
  }
  return res;
}

static void
ars_set_property (GObject * obj, guint id, const GValue * value, GParamSpec * pspec)
{
  GstCudaAudioResample *self = (GstCudaAudioResample *) obj;
  switch (id) {
    case PROP_QUALITY: self->quality = g_value_get_int (value); break;
    case PROP_DEVICE_ID: self->device_id = g_value_get_int (value); break;
    case PROP_RESAMPLE_METHOD: self->method = g_value_get_enum (value); break;
    case PROP_SINC_FILTER_MODE: self->sinc_filter_mode = g_value_get_enum (value); break;
    case PROP_SINC_FILTER_AUTO_THRESHOLD: self->sinc_filter_auto_threshold = g_value_get_uint (value); break;
    case PROP_SINC_FILTER_INTERPOLATION: self->sinc_filter_interpolation = g_value_get_enum (value); break;
    default: G_OBJECT_WARN_INVALID_PROPERTY_ID (obj, id, pspec); break;
  }
}

static void
ars_get_property (GObject * obj, guint id, GValue * value, GParamSpec * pspec)
{
  GstCudaAudioResample *self = (GstCudaAudioResample *) obj;
  switch (id) {
    case PROP_QUALITY: g_value_set_int (value, self->quality); break;
    case PROP_DEVICE_ID: g_value_set_int (value, self->device_id); break;
    case PROP_RESAMPLE_METHOD: g_value_set_enum (value, self->method); break;
    case PROP_SINC_FILTER_MODE: g_value_set_enum (value, self->sinc_filter_mode); break;
    case PROP_SINC_FILTER_AUTO_THRESHOLD: g_value_set_uint (value, self->sinc_filter_auto_threshold); break;
    case PROP_SINC_FILTER_INTERPOLATION: g_value_set_enum (value, self->sinc_filter_interpolation); break;
    default: G_OBJECT_WARN_INVALID_PROPERTY_ID (obj, id, pspec); break;
  }
}

static void
gst_cuda_audio_resample_class_init (GstCudaAudioResampleClass * klass)
{
  GObjectClass *gobject = G_OBJECT_CLASS (klass);
  GstElementClass *element = GST_ELEMENT_CLASS (klass);
  GstBaseTransformClass *trans = GST_BASE_TRANSFORM_CLASS (klass);
  gobject->set_property = ars_set_property;
  gobject->get_property = ars_get_property;
  g_object_class_install_property (gobject, PROP_QUALITY, g_param_spec_int ("quality", "Quality",
          "Resample quality with 0 being the lowest and 10 being the best", 0, 10, 4,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_DEVICE_ID, g_param_spec_int ("cuda-device-id", "Cuda Device ID",
          "GPU device to use", 0, G_MAXINT, 0, G_PARAM_READWRITE | GST_PARAM_MUTABLE_READY | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_RESAMPLE_METHOD, g_param_spec_enum ("resample-method", "Resample method to use",
          "What resample method to use", GST_TYPE_AUDIO_RESAMPLER_METHOD, GST_AUDIO_RESAMPLER_METHOD_KAISER,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_SINC_FILTER_MODE, g_param_spec_enum ("sinc-filter-mode", "Sinc filter table mode",
          "What sinc filter table mode to use", GST_TYPE_AUDIO_RESAMPLER_FILTER_MODE, GST_AUDIO_RESAMPLER_FILTER_MODE_AUTO,
          G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_SINC_FILTER_AUTO_THRESHOLD, g_param_spec_uint ("sinc-filter-auto-threshold",
          "Sinc filter auto mode threshold", "Memory usage threshold to use if sinc filter mode is AUTO, given in bytes "
          "(the stock resampler never sees it: SURVEY A.10)", 0, G_MAXUINT, 1 * 1048576, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  g_object_class_install_property (gobject, PROP_SINC_FILTER_INTERPOLATION, g_param_spec_enum ("sinc-filter-interpolation",
          "Sinc filter interpolation", "How to interpolate the sinc filter table", GST_TYPE_AUDIO_RESAMPLER_FILTER_INTERPOLATION,
          GST_AUDIO_RESAMPLER_FILTER_INTERPOLATION_CUBIC, G_PARAM_READWRITE | G_PARAM_STATIC_STRINGS));
  gst_element_class_add_static_pad_template (element, &ars_sink);
  gst_element_class_add_static_pad_template (element, &ars_src);
  gst_element_class_set_static_metadata (element, "CUDA audio resampler", "Filter/Converter/Audio/Hardware",
      "Bit-exact audioresample (F32, kaiser) polyphase FIR on sm_90a (libb200dsp)", "b200-gst-dsp");
  trans->start = ars_start;
  trans->stop = ars_stop;
  trans->get_unit_size = ars_get_unit_size;
  trans->transform_caps = ars_transform_caps;
  trans->transform_size = ars_transform_size;
  trans->set_caps = ars_set_caps;
  trans->transform = ars_transform;
  trans->sink_event = ars_sink_event;
  GST_DEBUG_CATEGORY_INIT (cuda_ars_debug, "cudaaudioresample", 0, "CUDA audio resampler");
}

static void
gst_cuda_audio_resample_init (GstCudaAudioResample * self)
{
  self->quality = 4;
  self->device_id = 0;
  self->method = GST_AUDIO_RESAMPLER_METHOD_KAISER;
  self->sinc_filter_mode = GST_AUDIO_RESAMPLER_FILTER_MODE_AUTO;
  self->sinc_filter_auto_threshold = 1 * 1048576;
  self->sinc_filter_interpolation = GST_AUDIO_RESAMPLER_FILTER_INTERPOLATION_CUBIC;
  self->t0 = GST_CLOCK_TIME_NONE;
  self->need_discont = TRUE;
}
