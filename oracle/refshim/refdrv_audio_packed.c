/* oracle/refshim/refdrv_audio_packed.c — TEST INFRASTRUCTURE ONLY.
 *
 * audioresample on a sample format its converter does not resample unconverted, composed from the reference's own
 * pieces in the order converter_generic runs them (gst-libs/gst/audio/audio-converter.c:1281-1310):
 *   finfo->unpack_func (..., GST_AUDIO_PACK_FLAG_TRUNCATE_RANGE, ...)          do_unpack :455-490 (silence when no input)
 *   gst_audio_resampler_resample in finfo->unpack_format                       chain_resample, do_resample
 *   gst_audio_quantize_samples (integer output narrower than 32 bits)          chain_quantize :968-1021
 *   finfo->pack_func (..., 0, ...)                                             :1305
 * The quantizer is created as chain_quantize creates it with the converter's defaults (dither none, noise shaping
 * none, :292-295; audioresample sets neither).  The resampler comes from ref_ars_new_opts (refdrv_audio.c), which
 * configures it as the element does; update / reset / get_out_frames go through ref_ars_* on ref_ars_packed_resampler.
 */
#include <gst/audio/audio.h>
#include <stdlib.h>
#include <string.h>
#include "audio-quantize.h"

GstAudioResampler *ref_ars_new_opts (int in_rate, int out_rate, int channels, int quality, int format, int method,
    int filter_mode, int interpolation);

typedef struct {
  GstAudioResampler *r;
  const GstAudioFormatInfo *finfo, *uinfo;
  GstAudioQuantize *quant;
  int channels;
} RefArsPacked;

RefArsPacked *
ref_ars_new_packed (int in_rate, int out_rate, int channels, int quality, int format, int method, int filter_mode,
    int interpolation)
{
  RefArsPacked *p = calloc (1, sizeof (*p));
  p->finfo = gst_audio_format_get_info ((GstAudioFormat) format);
  p->uinfo = gst_audio_format_get_info (p->finfo->unpack_format);
  p->channels = channels;
  p->r = ref_ars_new_opts (in_rate, out_rate, channels, quality, p->finfo->unpack_format, method, filter_mode,
      interpolation);
  if (GST_AUDIO_FORMAT_INFO_IS_INTEGER (p->finfo) && GST_AUDIO_FORMAT_INFO_DEPTH (p->finfo) < 32)
    p->quant = gst_audio_quantize_new (GST_AUDIO_DITHER_NONE, GST_AUDIO_NOISE_SHAPING_NONE, 0, GST_AUDIO_FORMAT_S32,
        channels, 1U << (32 - GST_AUDIO_FORMAT_INFO_DEPTH (p->finfo)));
  return p;
}

GstAudioResampler *
ref_ars_packed_resampler (RefArsPacked * p)
{
  return p->r;
}

void
ref_ars_free_packed (RefArsPacked * p)
{
  gst_audio_resampler_free (p->r);
  if (p->quant)
    gst_audio_quantize_free (p->quant);
  free (p);
}

size_t
ref_ars_process_packed (RefArsPacked * p, const void *in, size_t in_frames, void *out, size_t out_capacity)
{
  const size_t bps = GST_AUDIO_FORMAT_INFO_WIDTH (p->uinfo) / 8, ch = (size_t) p->channels;
  size_t n = gst_audio_resampler_get_out_frames (p->r, in_frames);
  gpointer tin = calloc (in_frames * ch + 1, bps), tout;
  gpointer ins[1] = { tin }, outs[1];
  if (n > out_capacity)
    n = out_capacity;
  tout = calloc (n * ch + 1, bps);
  outs[0] = tout;
  if (in)
    p->finfo->unpack_func (p->finfo, GST_AUDIO_PACK_FLAG_TRUNCATE_RANGE, tin, in, (gint) (in_frames * ch));
  else
    gst_audio_format_info_fill_silence (p->uinfo, tin, in_frames * ch * bps);
  gst_audio_resampler_resample (p->r, ins, in_frames, outs, n);
  if (p->quant)
    gst_audio_quantize_samples (p->quant, outs, outs, (guint) n);
  p->finfo->pack_func (p->finfo, 0, tout, out, (gint) (n * ch));
  free (tin);
  free (tout);
  return n;
}
