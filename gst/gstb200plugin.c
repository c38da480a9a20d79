/* gst/gstb200plugin.c — plugin entry of the CUDA raw-frame DSP elements.
 *
 * Exports gst_plugin_b200_get_desc / gst_plugin_b200_register through GST_PLUGIN_DEFINE
 * (gstreamer/gst/gstplugin.h:274-307) and registers the three elements the way
 * gst-plugins-bad/sys/nvcodec/plugin.c:950-956 registers the stock CUDA ones.
 * Builds only where GStreamer >= 1.22 + libgstcuda are installed (gst/meson.build).
 */
#include <gst/gst.h>

#include "gstb200elements.h"

static gboolean
plugin_init (GstPlugin * plugin)
{
  gboolean ok = TRUE;

  /* rank NONE: opt-in drop-ins, selected explicitly in the pipeline description */
  ok &= gst_element_register (plugin, "cudavideoconvertscale", GST_RANK_NONE,
      GST_TYPE_CUDA_VIDEO_CONVERT_SCALE);
  ok &= gst_element_register (plugin, "cudacompositor", GST_RANK_NONE, GST_TYPE_B200_CUDA_COMPOSITOR);
  ok &= gst_element_register (plugin, "cudaaudioresample", GST_RANK_NONE, GST_TYPE_CUDA_AUDIO_RESAMPLE);
  return ok;
}

GST_PLUGIN_DEFINE (GST_VERSION_MAJOR, GST_VERSION_MINOR, b200,
    "CUDA colourspace/scale, compositor and audio resampler (libb200dsp)",
    plugin_init, VERSION, "LGPL", PACKAGE, "https://example.invalid/gst-b200")
