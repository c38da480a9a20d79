/* declarations only: gst-plugins-base/gst-libs/gst/audio/audio-info.h, audio-format.h, audio-resampler.h */
#ifndef B200_STUB_AUDIO_H
#define B200_STUB_AUDIO_H
#include <gst/gst.h>
typedef enum { GST_AUDIO_FORMAT_UNKNOWN = 0 } GstAudioFormat;
typedef struct { GstAudioFormat format; } GstAudioFormatInfo;
typedef struct _GstAudioInfo { const GstAudioFormatInfo *finfo; guint flags; gint layout, rate, channels, bpf; } GstAudioInfo;
#define GST_AUDIO_INFO_RATE(i) ((i)->rate)
#define GST_AUDIO_INFO_CHANNELS(i) ((i)->channels)
#define GST_AUDIO_INFO_BPF(i) ((i)->bpf)
#define GST_AUDIO_INFO_FORMAT(i) ((i)->finfo->format)
#define GST_AUDIO_NE(s) #s "LE"
#define GST_AUDIO_FORMATS_ALL "{ F64LE, F64BE, F32LE, F32BE, S32LE, S32BE, U32LE, U32BE, S24_32LE, S24_32BE, U24_32LE, " \
    "U24_32BE, S24LE, S24BE, U24LE, U24BE, S20_32LE, S20_32BE, U20_32LE, U20_32BE, S20LE, S20BE, U20LE, U20BE, S18LE, " \
    "S18BE, U18LE, U18BE, S16LE, S16BE, U16LE, U16BE, S8, U8 }"
gboolean gst_audio_info_from_caps (GstAudioInfo * info, const GstCaps * caps);
enum { GST_AUDIO_RESAMPLER_METHOD_NEAREST, GST_AUDIO_RESAMPLER_METHOD_LINEAR, GST_AUDIO_RESAMPLER_METHOD_CUBIC,
  GST_AUDIO_RESAMPLER_METHOD_BLACKMAN_NUTTALL, GST_AUDIO_RESAMPLER_METHOD_KAISER };
enum { GST_AUDIO_RESAMPLER_FILTER_MODE_INTERPOLATED, GST_AUDIO_RESAMPLER_FILTER_MODE_FULL, GST_AUDIO_RESAMPLER_FILTER_MODE_AUTO };
enum { GST_AUDIO_RESAMPLER_FILTER_INTERPOLATION_NONE, GST_AUDIO_RESAMPLER_FILTER_INTERPOLATION_LINEAR, GST_AUDIO_RESAMPLER_FILTER_INTERPOLATION_CUBIC };
GType gst_audio_resampler_method_get_type (void); GType gst_audio_resampler_filter_mode_get_type (void);
GType gst_audio_resampler_filter_interpolation_get_type (void);
#define GST_TYPE_AUDIO_RESAMPLER_METHOD (gst_audio_resampler_method_get_type ())
#define GST_TYPE_AUDIO_RESAMPLER_FILTER_MODE (gst_audio_resampler_filter_mode_get_type ())
#define GST_TYPE_AUDIO_RESAMPLER_FILTER_INTERPOLATION (gst_audio_resampler_filter_interpolation_get_type ())
#endif
