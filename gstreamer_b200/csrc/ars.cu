// gstreamer_b200/csrc/ars.cu — b200_ars_* : polyphase FIR audio resampler (product code, sm_90a).
//
// Replaces, for F32 interleaved audio with the audioresample element's defaults
// (kaiser, filter-mode auto, cubic filter interpolation; gst/audioresample/gstaudioresample.c:68-72):
//   gst_audio_resampler_new / update / calculate_taps   gst-libs/gst/audio/audio-resampler.c:1344, :1502, :1062
//   get_taps_gfloat_full (phase cache)                  audio-resampler.c:503-561
//   resample_gfloat_full_1_sse + inner product          audio-resampler-macros.h:62-100, audio-resampler-x86-sse.c:27-46
//   framing: get_out_frames / resample                  audio-resampler.c:1648-1678, :1750-1805
//
// Device side: one thread = one channel (lanes = 32 adjacent channels, so every load/store of
// the interleaved stream is a fully coalesced 128 B row) x RQ consecutive output frames whose
// input windows overlap by >90 %, so each input sample is loaded once per thread and feeds RQ
// accumulator sets.  Bit-exactness with the reference's SSE kernel comes from keeping its lane
// structure: four partial sums by (tap index mod 4), separate multiply and add (no FMA), final
// (l0+l2)+(l1+l3).  Indexing the partial sums by the ABSOLUTE input index mod 4 instead of the
// tap index only rotates the lanes, and the final reduction is invariant under rotation.
// Tap rows are staged per CTA in shared memory pre-shifted to the window alignment of each
// output so that all tap loads are aligned 128-bit broadcasts.
#include "common.h"
#ifndef B200_CUDA_EMU
#include <cuda.h>            // CUtensorMap types only: the encoder is fetched through cudaGetDriverEntryPoint
#endif

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include <algorithm>
#include <vector>

#include "besi0_coeffs.inc"

namespace b200 {

// ------------------------------------------------------------------------------ host: filter design
static double bessel_i0 (double x)
{
  const double w = fabs (x);
  double t, y;
  if (w < 8.5) {
    t = w * w * 0.0625;
    const double *p = B200_I0_LOW + 13 * (int) t;
    y = p[0];
    for (int i = 1; i < 13; i++) y = y * t + p[i];
  } else if (w < 12.5) {
    const int k = (int) w;
    t = w - k;
    const double *p = B200_I0_MID + 14 * (k - 8);
    y = p[0];
    for (int i = 1; i < 14; i++) y = y * t + p[i];
  } else {
    t = 60 / w;
    const double *p = B200_I0_HIGH + 9 * (int) t;
    y = p[0];
    for (int i = 1; i < 9; i++) y = y * t + p[i];
    y = y * sqrt (t) * exp (w);
  }
  return y;
}

// The caller's samples of a format the resampler does not work in (converter_generic, audio-converter.c:1281-1310): each
// is unpacked on load (do_unpack with GST_AUDIO_PACK_FLAG_TRUNCATE_RANGE, :455-490) and quantized and packed on store
// (chain_quantize :968-1021, pack flags 0 :1305).  Warp-uniform: one descriptor per launch.
enum ArsIoKind : int { ARS_IO_NONE = 0, ARS_IO_INT = 1, ARS_IO_F32 = 2, ARS_IO_F64 = 3 };
struct ArsIo {
  int kind;                      // ArsIoKind: integer -> S32, F32BE -> F64, F64BE -> F64
  int step;                      // bytes from one sample to the next
  int big;                       // big-endian bytes
  int shift;                     // integer formats: 32 - depth (unpack shifts left, pack right)
  int arith;                     // pack shifts arithmetically (signed 4-byte formats: shrsl of pack_s24_32)
  int qshift;                    // quantize to depth bits (32 - depth) or 0 (32-bit formats)
  unsigned sign;                 // 0x80000000 for unsigned formats
};

struct ArsPlan {
  int channels = 0, in_step = 0, out_step = 0;   // rates / gcd
  int samp_inc = 0, samp_frac = 0;
  int n_taps = 0, oversample = 0, n_phases = 0;
  bool full = false;
  bool blackman = false;         // resample-method=blackman-nuttall (else kaiser)
  bool copy = false;             // equal rates: the reference selects its nearest functions (setup_functions :1019-1020)
  int small = 0;                 // resample-method nearest (1) / linear (2) / cubic (3): a few taps, no sinc table, FULL mode
  bool linear = false;           // sinc-filter-interpolation=linear: two prototype rows per phase, 11x the oversampling
  int isize = 4;                 // prototype rows one phase reads (4 cubic, 2 linear)
  bool interp_none = false;      // FULL mode with sinc-filter-interpolation=none: every phase's taps computed directly
  double cutoff = 0, beta = 0;
  std::vector<float> proto;      // (oversample + isize) x n_taps oversampled prototype
  std::vector<float> phases;     // n_phases x n_taps (FULL mode), all phases precomputed
  // other sample formats: the same two tables in the samples' own type
  int fmt = 0, bps = 4;          // ArsFmt, bytes per sample: the format the resampler works in, and its history holds
  std::vector<uint8_t> proto_x, phases_x;
  ArsIo io = ArsIo ();           // how the caller's samples are stored (io.kind == ARS_IO_NONE: as fmt)
  int width = 4;                 // bytes per sample in the caller's buffers
};

enum ArsFmt : int { ARS_F32 = 0, ARS_S16 = 1, ARS_S32 = 2, ARS_F64 = 3 };

// Every GstAudioFormat (audio-format.c formats[], :249-418): packed width and step in bytes, depth, signedness, byte order,
// float.  The step differs from the width only in the 20-bit _32 formats, whose pack / unpack functions are the 3-byte
// ones (MAKE_PACK_UNPACK (s20_32le, 3, ...), audio-format.c:206-213).  Integer formats unpack to S32 and float formats to
// F64 (their unpack_format); the quantize shift of an integer format is 32 - depth.
static const struct ArsFormatInfo { int format, width, step, depth; bool is_signed, big, is_float; } kArsFormats[] = {
  {B200_AUDIO_FORMAT_S8, 1, 1, 8, true, false, false},           {B200_AUDIO_FORMAT_U8, 1, 1, 8, false, false, false},
  {B200_AUDIO_FORMAT_S16LE, 2, 2, 16, true, false, false},       {B200_AUDIO_FORMAT_S16BE, 2, 2, 16, true, true, false},
  {B200_AUDIO_FORMAT_U16LE, 2, 2, 16, false, false, false},      {B200_AUDIO_FORMAT_U16BE, 2, 2, 16, false, true, false},
  {B200_AUDIO_FORMAT_S24_32LE, 4, 4, 24, true, false, false},    {B200_AUDIO_FORMAT_S24_32BE, 4, 4, 24, true, true, false},
  {B200_AUDIO_FORMAT_U24_32LE, 4, 4, 24, false, false, false},   {B200_AUDIO_FORMAT_U24_32BE, 4, 4, 24, false, true, false},
  {B200_AUDIO_FORMAT_S32LE, 4, 4, 32, true, false, false},       {B200_AUDIO_FORMAT_S32BE, 4, 4, 32, true, true, false},
  {B200_AUDIO_FORMAT_U32LE, 4, 4, 32, false, false, false},      {B200_AUDIO_FORMAT_U32BE, 4, 4, 32, false, true, false},
  {B200_AUDIO_FORMAT_S24LE, 3, 3, 24, true, false, false},       {B200_AUDIO_FORMAT_S24BE, 3, 3, 24, true, true, false},
  {B200_AUDIO_FORMAT_U24LE, 3, 3, 24, false, false, false},      {B200_AUDIO_FORMAT_U24BE, 3, 3, 24, false, true, false},
  {B200_AUDIO_FORMAT_S20LE, 3, 3, 20, true, false, false},       {B200_AUDIO_FORMAT_S20BE, 3, 3, 20, true, true, false},
  {B200_AUDIO_FORMAT_U20LE, 3, 3, 20, false, false, false},      {B200_AUDIO_FORMAT_U20BE, 3, 3, 20, false, true, false},
  {B200_AUDIO_FORMAT_S18LE, 3, 3, 18, true, false, false},       {B200_AUDIO_FORMAT_S18BE, 3, 3, 18, true, true, false},
  {B200_AUDIO_FORMAT_U18LE, 3, 3, 18, false, false, false},      {B200_AUDIO_FORMAT_U18BE, 3, 3, 18, false, true, false},
  {B200_AUDIO_FORMAT_F32LE, 4, 4, 32, true, false, true},        {B200_AUDIO_FORMAT_F32BE, 4, 4, 32, true, true, true},
  {B200_AUDIO_FORMAT_F64LE, 8, 8, 64, true, false, true},        {B200_AUDIO_FORMAT_F64BE, 8, 8, 64, true, true, true},
  {B200_AUDIO_FORMAT_S20_32LE, 4, 3, 20, true, false, false},    {B200_AUDIO_FORMAT_S20_32BE, 4, 3, 20, true, true, false},
  {B200_AUDIO_FORMAT_U20_32LE, 4, 3, 20, false, false, false},   {B200_AUDIO_FORMAT_U20_32BE, 4, 3, 20, false, true, false},
};

// convert_taps_gint16_c / _gint32_c (audio-resampler.c:217-258): round with a bias found by bisection so that
// the integer taps sum to (1 << precision) - 1
template <typename T>
static void convert_taps_int (const double *tmp, T *taps, double weight, int n, int precision)
{
  const long long one = (1LL << precision) - 1;
  const double multiplier = (double) one;
  double offset = 0.5, l_offset = 0.0, h_offset = 1.0;
  for (int i = 0; i < 32; i++) {
    long long sum = 0;
    for (int j = 0; j < n; j++) sum += (long long) floor (offset + tmp[j] * multiplier / weight);
    if (sum == one || l_offset == h_offset) break;
    if (sum < one) { if (offset > l_offset) l_offset = offset; offset += (h_offset - l_offset) / 2; }
    else { if (offset < h_offset) h_offset = offset; offset -= (h_offset - l_offset) / 2; }
  }
  for (int j = 0; j < n; j++) taps[j] = (T) floor (offset + tmp[j] * multiplier / weight);
}

// make_coeff_gint16_cubic / make_coeff_gint32_cubic (audio-resampler.c:350-372); host and device
__host__ __device__ inline void cubic_coeff_s16 (int num, int denom, int ic[4])
{
  const int x = (int) (((long long) num << 15) / denom);
  const int x2 = (int) ((unsigned) x * (unsigned) x) >> 15, x3 = (int) ((unsigned) x2 * (unsigned) x) >> 15;
  const short c0 = (short) ((((x3 - x) * 32768) / 6) >> 15);      // (a << 15) of the reference, without shifting a negative value
  const short c1 = (short) (x + ((x2 - x3) >> 1));
  const short c3 = (short) (-(((x * 32768) / 3) >> 15) + (x2 >> 1) - (((x3 * 32768) / 6) >> 15));
  ic[0] = c0; ic[1] = c1; ic[3] = c3;
  ic[2] = (short) (32767 - c0 - c1 - c3);
}
__host__ __device__ inline void cubic_coeff_s32 (int num, int denom, int ic[4])
{
  const long long one = (1LL << 31) - 1;
  const long long x = ((long long) num << 31) / denom, x2 = (x * x) >> 31, x3 = (x2 * x) >> 31;
  ic[0] = (int) ((((x3 - x) * (1LL << 31)) / 6) >> 31);
  ic[1] = (int) (x + ((x2 - x3) >> 1));
  ic[3] = (int) (-(((x * (1LL << 31)) / 3) >> 31) + (x2 >> 1) - (((x3 * (1LL << 31)) / 6) >> 31));
  ic[2] = (int) (one - ic[0] - ic[1] - ic[3]);
}
// make_coeff_gdouble_cubic: float literals promoted to double; no FMA may be formed
static void cubic_coeff_f64_host (int num, int denom, double ic[4])
{
  volatile double x = (double) num / denom, x2 = x * x, x3 = x2 * x;
  volatile double a = x3 - x, b = x2 - x3, c = 0.5f * b;
  ic[0] = 0.16667f * a;
  ic[1] = x + c;
  volatile double d = -0.33333f * x, e = 0.5f * x2, f = 0.16667f * x3, g = d + e;
  ic[3] = g - f;
  volatile double h = (double) 1.0 - ic[0], k = h - ic[1];
  ic[2] = k - ic[3];
}


static const struct { double cutoff, down, atten, trbw; } kKaiser[11] = {
  {0.860, 0.96511, 60, 0.7}, {0.880, 0.96591, 65, 0.29}, {0.910, 0.96923, 70, 0.145},
  {0.920, 0.97600, 80, 0.105}, {0.940, 0.97979, 85, 0.087}, {0.940, 0.98085, 95, 0.077},
  {0.945, 0.99471, 100, 0.068}, {0.950, 1.0, 105, 0.055}, {0.960, 1.0, 110, 0.045},
  {0.968, 1.0, 115, 0.039}, {0.975, 1.0, 120, 0.0305}
};
static const int kOversample[11] = {4, 4, 4, 8, 8, 16, 16, 16, 16, 32, 32};

static void cubic_coeff (int num, int denom, float ic[4])
{
  // make_coeff_gfloat_cubic (audio-resampler.c:360-373): float arithmetic, these literals
  const float x = (float) num / denom, x2 = x * x, x3 = x2 * x;
  ic[0] = 0.16667f * (x3 - x);
  ic[1] = x + 0.5f * (x2 - x3);
  ic[3] = -0.33333f * x + 0.5f * x2 - 0.16667f * x3;
  ic[2] = (float) 1.0 - ic[0] - ic[1] - ic[3];
}

// forced_div > 0: the divisor gst_audio_resampler_update () settled on (a rate change keeps the common divisor only as far
// as the rescaled phase allows, audio-resampler.c:1525-1551); 0: the plain gcd of a fresh resampler
static int build_ars_plan (const b200_ars_config & cfg, ArsPlan * p, int forced_div = 0)
{
  if (cfg.in_rate <= 0 || cfg.out_rate <= 0 || cfg.channels <= 0 || cfg.quality < 0 || cfg.quality > 10)
    return B200_ERR_INVALID_ARG;
  switch (cfg.format) {          // GstAudioFormat values, native endianness (audio-format.h:97-140)
    case 0: case B200_AUDIO_FORMAT_F32LE: p->fmt = ARS_F32; p->bps = 4; break;
    case B200_AUDIO_FORMAT_S16LE: p->fmt = ARS_S16; p->bps = 2; break;
    case B200_AUDIO_FORMAT_S32LE: p->fmt = ARS_S32; p->bps = 4; break;
    case B200_AUDIO_FORMAT_F64LE: p->fmt = ARS_F64; p->bps = 8; break;
    default: {                   // unpacked to the format's unpack_format
      const ArsFormatInfo *f = nullptr;
      for (const ArsFormatInfo & e : kArsFormats) if (e.format == cfg.format) f = &e;
      if (!f) return B200_ERR_UNSUPPORTED;
      p->fmt = f->is_float ? ARS_F64 : ARS_S32;
      p->bps = f->is_float ? 8 : 4;
      p->io.kind = !f->is_float ? ARS_IO_INT : (f->width == 4 ? ARS_IO_F32 : ARS_IO_F64);
      p->io.step = f->step;
      p->io.big = f->big;
      p->io.shift = f->is_float ? 0 : 32 - f->depth;
      p->io.arith = f->is_signed && f->step == 4;
      p->io.qshift = f->is_float ? 0 : 32 - f->depth;
      p->io.sign = f->is_signed ? 0u : 0x80000000u;
      p->width = f->width;
    }
  }
  if (p->io.kind == ARS_IO_NONE) p->width = p->bps;
  p->channels = cfg.channels;
  int a = cfg.in_rate, b = cfg.out_rate;
  while (b) { int t = a; a = b; b = t % b; }
  if (forced_div > 0) a = forced_div;
  p->in_step = cfg.in_rate / a;
  p->out_step = cfg.out_rate / a;
  p->samp_inc = p->in_step / p->out_step;
  p->samp_frac = p->in_step % p->out_step;
  const auto & q = kKaiser[cfg.quality];
  double fc = q.cutoff;
  if (cfg.out_rate < cfg.in_rate) fc *= q.down;
  const double A = q.atten;
  p->beta = A > 50 ? 0.1102 * (A - 8.7) : (A >= 21 ? 0.5842 * pow (A - 21, 0.4) + 0.07886 * (A - 21) : 0.0);
  const double dw = 2 * M_PI * q.trbw;
  p->n_taps = (int) ((A - 8.0) / (2.285 * dw)) + 1;
  p->cutoff = fc;
  // the element's other properties: only what needs no new device code - both windowed-sinc methods, every filter
  // mode, and every table interpolation
  if (cfg.resample_method < 0 || cfg.resample_method > B200_ARS_METHOD_KAISER) return B200_ERR_INVALID_ARG;
  // nearest / linear / cubic run in their own small kernel (ars_small_kernel)
  if (cfg.resample_method >= B200_ARS_METHOD_NEAREST && cfg.resample_method <= B200_ARS_METHOD_CUBIC)
    p->small = cfg.resample_method;
  // equal rates (the element itself goes pass-through, gstaudioresample.c set_caps): every output is the first sample of
  // its window, through the same small kernel
  p->copy = p->in_step == p->out_step;
  if (cfg.sinc_filter_mode < 0 || cfg.sinc_filter_mode > B200_ARS_FILTER_MODE_AUTO) return B200_ERR_INVALID_ARG;
  if (cfg.sinc_filter_interpolation < 0 || cfg.sinc_filter_interpolation > B200_ARS_FILTER_INTERPOLATION_CUBIC)
    return B200_ERR_INVALID_ARG;
  p->blackman = cfg.resample_method == B200_ARS_METHOD_BLACKMAN_NUTTALL;
  if (p->blackman) {                    // blackman_qualities, audio-resampler.c:81-93; options_set_quality :1299-1305
    static const struct { int n_taps; double cutoff; } kBlackman[11] = {{8, 0.5}, {16, 0.6}, {24, 0.72}, {32, 0.8},
      {48, 0.85}, {64, 0.90}, {80, 0.92}, {96, 0.933}, {128, 0.950}, {148, 0.955}, {160, 0.960}};
    p->n_taps = kBlackman[cfg.quality].n_taps;
    p->cutoff = kBlackman[cfg.quality].cutoff;
  }
  // the methods without a sinc table (resampler_calculate_taps :1070-1117): 2 taps (nearest, never scaled), 2 (linear),
  // 4 (cubic, options_set_quality :1286-1297), not rounded up to 8; FULL mode with no table interpolation
  if (p->small) p->n_taps = p->small == B200_ARS_METHOD_CUBIC ? 4 : 2;
  const bool no_interp = p->small || cfg.sinc_filter_interpolation == B200_ARS_FILTER_INTERPOLATION_NONE;
  if (p->out_step < p->in_step && p->small != B200_ARS_METHOD_NEAREST) {
    p->cutoff = p->cutoff * p->out_step / p->in_step;
    p->n_taps = (int) (((unsigned long long) p->n_taps * p->in_step) / p->out_step);
  }
  if (!p->small) p->n_taps = (p->n_taps + 7) & ~7;
  int over = kOversample[cfg.quality];
  for (int mult = 2; over > 1 && mult * p->out_step < p->in_step; mult *= 2) over >>= 1;
  if (no_interp) over = 1;              // audio-resampler.c:1141-1143
  p->linear = !p->small && cfg.sinc_filter_interpolation == B200_ARS_FILTER_INTERPOLATION_LINEAR;
  if (p->linear) over *= 11;            // :1131-1137
  p->isize = p->linear ? 2 : 4;         // :1186-1197
  const int isize = p->isize;
  p->oversample = over;
  // filter-mode auto with the element's VARIABLE_RATE flag: FULL when the whole phase table is
  // below the (effectively fixed) 1 MiB threshold (audio-resampler.c:1147-1166)
  if (p->small)
    p->full = true;
  else if (cfg.sinc_filter_mode == 0 || cfg.sinc_filter_mode == B200_ARS_FILTER_MODE_AUTO)
    p->full = (long long) p->bps * p->n_taps * p->out_step < 1048576;     // bps * n_taps * out_rate, :1153
  else
    p->full = cfg.sinc_filter_mode == B200_ARS_FILTER_MODE_FULL;
  // an interpolated table with no interpolation falls back to the default cubic one, at the oversampling of 1 chosen
  // above (:1167-1170)
  p->interp_none = p->full && no_interp;
  p->n_phases = p->full ? p->out_step : 0;

  const int n = p->n_taps;
  p->proto.assign ((size_t) (over + isize) * n, 0.f);
  if (p->fmt != ARS_F32) p->proto_x.assign ((size_t) (over + isize) * n * p->bps, 0);
  std::vector<double> tmp (n);
  // make_taps (audio-resampler.c:287-323): n windowed-sinc values starting at x0, normalised, in float and (other
  // sample formats) in the samples' own type
  auto make_row = [&] (double x0, float *rowf, uint8_t *px) {
    double weight = 0.0;
    for (int i = 0; i < n; i++) {
      const double x = x0 + i, y = M_PI * x;
      const double s = (y == 0.0 ? p->cutoff : sin (y * p->cutoff) / y);
      if (p->small == B200_ARS_METHOD_LINEAR) {            // get_linear_tap, :163-168
        tmp[i] = ((n + 1) & ~1) / 2 - fabs (x);
      } else if (p->small == B200_ARS_METHOD_CUBIC) {      // get_cubic_tap :170-190, b = 1, c = 0 (:97-98)
        const double b = 1.0, c = 0.0, a = fabs (x * 4.0) / n, a2 = a * a, a3 = a2 * a;
        if (a <= 1.0) tmp[i] = ((12.0 - 9.0 * b - 6.0 * c) * a3 + (-18.0 + 12.0 * b + 6.0 * c) * a2 + (6.0 - 2.0 * b)) / 6.0;
        else if (a <= 2.0) tmp[i] = ((-b - 6.0 * c) * a3 + (6.0 * b + 30.0 * c) * a2 + (-12.0 * b - 48.0 * c) * a + (8.0 * b + 24.0 * c)) / 6.0;
        else tmp[i] = 0.0;
      } else if (p->blackman) {            // get_blackman_nuttall_tap, :192-203
        const double w = 2.0 * y / n + M_PI;
        tmp[i] = s * (0.3635819 - 0.4891775 * cos (w) + 0.1365995 * cos (2 * w) - 0.0106411 * cos (3 * w));
      } else {                             // get_kaiser_tap, :205-215
        const double w = 2.0 * x / n;
        tmp[i] = s * bessel_i0 (p->beta * sqrt (fmax (1 - w * w, 0)));
      }
      weight += tmp[i];
    }
    if (rowf) for (int i = 0; i < n; i++) rowf[i] = (float) (tmp[i] / weight);
    if (!px) return;
    if (p->fmt == ARS_S16) convert_taps_int (tmp.data (), (int16_t *) px, weight, n, 15);
    else if (p->fmt == ARS_S32) convert_taps_int (tmp.data (), (int32_t *) px, weight, n, 31);
    else if (p->fmt == ARS_F64) for (int i = 0; i < n; i++) ((double *) px)[i] = tmp[i] / weight;
  };
  // (the reference builds this table only with a table interpolation, :1181-1201; the small methods have none, and
  // their tap shapes can sum to zero on rows nobody would read)
  if (!p->small)
  for (int row = 0; row < over + isize; row++)
    make_row (-(n / 2) + row / (double) over, &p->proto[(size_t) row * n],
        p->fmt != ARS_F32 ? p->proto_x.data () + (size_t) row * n * p->bps : nullptr);
  if (p->small == B200_ARS_METHOD_NEAREST) {
    // no taps at all (make_taps :294-295, n_phases stays 0): one zero row so that the tables are never empty
    p->n_phases = 0;
    if (p->fmt == ARS_F32) p->phases.assign ((size_t) n, 0.f);
    else p->phases_x.assign ((size_t) n * p->bps, 0);
    return B200_OK;
  }
  if (p->interp_none) {
    // GST_AUDIO_RESAMPLER_FILTER_INTERPOLATION_NONE in FULL mode (get_taps_<type>_full :517-525): x = 1 - n/2 - phase/n_phases
    if (p->fmt == ARS_F32) p->phases.assign ((size_t) p->n_phases * n, 0.f);
    else p->phases_x.assign ((size_t) p->n_phases * n * p->bps, 0);
    for (int ph = 0; ph < p->n_phases; ph++)
      make_row (1.0 - n / 2 - (double) ph / p->n_phases, p->fmt == ARS_F32 ? &p->phases[(size_t) ph * n] : nullptr,
          p->fmt != ARS_F32 ? p->phases_x.data () + (size_t) ph * n * p->bps : nullptr);
    return B200_OK;
  }
  if (p->full && p->fmt != ARS_F32) {
    // every phase (get_taps_<type>_full): interpolate_gint16_cubic_sse2 / interpolate_gint32_cubic_c /
    // interpolate_gdouble_cubic_sse2 between four prototype rows
    p->phases_x.assign ((size_t) p->n_phases * n * p->bps, 0);
    for (int ph = 0; ph < p->n_phases; ph++) {
      const int pos = ph * over, offset = (over - 1) - pos / p->n_phases, frac = pos % p->n_phases;
      const uint8_t *c0 = p->proto_x.data () + (size_t) offset * n * p->bps;
      uint8_t *res = p->phases_x.data () + (size_t) ph * n * p->bps;
      if (p->linear && p->fmt == ARS_S16) {      // interpolate_gint16_linear_sse2 (audio-resampler-x86-sse2.c:267-299)
        const int x = (int) (((long long) frac << 15) / p->n_phases), y = 32767 - x;   // make_coeff_gint16_linear :325-332
        const int16_t *a = (const int16_t *) c0, *b = a + n;
        for (int i = 0; i < n; i++) {
          const int t = (int) ((unsigned) (a[i] * x) + (unsigned) (b[i] * y) + (1u << 14)) >> 15;
          ((int16_t *) res)[i] = (int16_t) (t < -32768 ? -32768 : (t > 32767 ? 32767 : t));
        }
      } else if (p->linear && p->fmt == ARS_S32) {   // interpolate_gint32_linear_c (audio-resampler.c:375-390); the store truncates
        const long long x = ((long long) frac << 31) / p->n_phases;
        const int32_t *a = (const int32_t *) c0, *b = a + n;
        for (int i = 0; i < n; i++) {
          const unsigned long long t = (unsigned long long) (((long long) a[i] - (long long) b[i]) * x) +
              ((unsigned long long) (long long) b[i] << 31);
          ((int32_t *) res)[i] = (int32_t) (uint32_t) ((long long) (t + (1ULL << 30)) >> 31);
        }
      } else if (p->linear) {                    // interpolate_gdouble_linear_sse2 (audio-resampler-x86-sse2.c:344-366)
        volatile double x = (double) frac / p->n_phases, y = 1.0 - x;
        const double *a = (const double *) c0, *b = a + n;
        for (int i = 0; i < n; i++) {
          volatile double t0 = a[i] * x, t1 = b[i] * y;
          ((double *) res)[i] = t0 + t1;
        }
      } else if (p->fmt == ARS_S16) {
        int ic[4];
        cubic_coeff_s16 (frac, p->n_phases, ic);
        const int16_t *a = (const int16_t *) c0, *b = a + n, *c = b + n, *d = c + n;
        for (int i = 0; i < n; i++) {
          const int t = (int) ((unsigned) (a[i] * ic[0]) + (unsigned) (b[i] * ic[1]) + (unsigned) (c[i] * ic[2]) +
              (unsigned) (d[i] * ic[3]) + (1u << 14)) >> 15;
          ((int16_t *) res)[i] = (int16_t) (t < -32768 ? -32768 : (t > 32767 ? 32767 : t));
        }
      } else if (p->fmt == ARS_S32) {
        int ic[4];
        cubic_coeff_s32 (frac, p->n_phases, ic);
        const int32_t *a = (const int32_t *) c0, *b = a + n, *c = b + n, *d = c + n;
        for (int i = 0; i < n; i++) {
          long long t = (long long) a[i] * ic[0] + (long long) b[i] * ic[1] + (long long) c[i] * ic[2] + (long long) d[i] * ic[3];
          t = (t + (1LL << 30)) >> 31;
          ((int32_t *) res)[i] = (int32_t) (t < -(1LL << 31) ? -(1LL << 31) : (t > (1LL << 31) - 1 ? (1LL << 31) - 1 : t));
        }
      } else {
        double ic[4];
        cubic_coeff_f64_host (frac, p->n_phases, ic);
        const double *a = (const double *) c0, *b = a + n, *c = b + n, *d = c + n;
        for (int i = 0; i < n; i++) {
          volatile double t0 = a[i] * ic[0], t1 = b[i] * ic[1], t2 = c[i] * ic[2], t3 = d[i] * ic[3];
          volatile double u0 = t0 + t1, u2 = t2 + t3;
          ((double *) res)[i] = u0 + u2;
        }
      }
    }
  }
  if (p->fmt != ARS_F32) return B200_OK;
  if (p->full) {
    // every phase, built exactly as the reference builds it lazily (get_taps_gfloat_full +
    // interpolate_gfloat_cubic_sse: (c0*f0 + c1*f1) + (c2*f2 + c3*f3))
    p->phases.assign ((size_t) p->n_phases * n, 0.f);
    for (int ph = 0; ph < p->n_phases; ph++) {
      const int pos = ph * over, offset = (over - 1) - pos / p->n_phases, frac = pos % p->n_phases;
      float ic[4];
      const float *c0 = &p->proto[(size_t) offset * n], *c1 = c0 + n, *c2 = c1 + n, *c3 = c2 + n;
      float *res = &p->phases[(size_t) ph * n];
      if (p->linear) {          // make_coeff_gfloat_linear (:333-340) + interpolate_gfloat_linear_sse: c0*f0 + c1*f1
        volatile float x = (float) frac / p->n_phases, y = 1.0f - x;
        for (int i = 0; i < n; i++) {
          volatile float t0 = c0[i] * x, t1 = c1[i] * y;
          res[i] = t0 + t1;
        }
        continue;
      }
      cubic_coeff (frac, p->n_phases, ic);
      for (int i = 0; i < n; i++) {
        volatile float t0 = c0[i] * ic[0], t1 = c1[i] * ic[1], t2 = c2[i] * ic[2], t3 = c3[i] * ic[3];
        volatile float u0 = t0 + t1, u2 = t2 + t3;
        res[i] = u0 + u2;
      }
    }
  }
  return B200_OK;
}

// ------------------------------------------------------------------------------ device
constexpr int ARS_RQ = 4;        // output frames per thread pass
constexpr int ARS_THREADS = 256;
constexpr int ARS_TILE_SMEM = 110 * 1024;   // dynamic shared memory the tile kernel may ask for (2 CTAs/SM)

struct ArsLaunch {
  const float *hist;             // [hist_frames][channels] retained input
  const float *in;               // [in_frames][channels] or nullptr (silence)
  float *out;
  const float *phases;           // [n_phases][n_taps]
  long long hist_frames, avail;  // avail = hist_frames + in_frames
  long long out_frames;
  int channels, n_taps, out_step, samp_inc, samp_frac;
  int samp_index, samp_phase;    // state at the start of this call
  int no;                        // output frames per CTA (multiple of ARS_RQ)
  int wcn;                       // warps across channels
  int row_pitch;                 // floats per staged tap row (multiple of 4)
};

__device__ __forceinline__ void ars_position (const ArsLaunch & L, long long o, long long &idx, int &phase)
{
  // closed form of the per-sample stepping in get_taps_* (audio-resampler.c:554-559)
  const long long t = (long long) L.samp_phase + o * L.samp_frac;
  idx = (long long) L.samp_index + o * L.samp_inc + t / L.out_step;
  phase = (int) (t % L.out_step);
}

// the samples of stream frame f: a row of the retained history, a row of the caller's input, or nullptr (silence)
template <typename T>
__device__ __forceinline__ const T *ars_frame_row (const ArsLaunch & L, long long f)
{
  const T *src = nullptr;
  if (f < L.hist_frames) src = (const T *) L.hist + f * L.channels;
  else if (f < L.avail && L.in) src = (const T *) L.in + (f - L.hist_frames) * L.channels;
  return src;
}

// (l0 + l2) + (l1 + l3): the final reduction of the four partial sums, audio-resampler-x86-sse.c:43-45
__device__ __forceinline__ float ars_lane_sum (const float l[4])
{
  return __fadd_rn (__fadd_rn (l[0], l[2]), __fadd_rn (l[1], l[3]));
}

// The F32 inner products of one group of RQ consecutive outputs for CPT adjacent channels over a staged [frame][CB]
// window: xp = the thread's first channel at the group's first (chunk-aligned) frame, tp = the group's chunk-major taps
// (RQ float4 per chunk), nch chunks.  Four partial sums per (channel, output) by tap index mod 4, separate multiply and
// add (no FMA); ars_lane_sum reduces them.
template <int CPT, int CB>
__device__ __forceinline__ void ars_group_f32 (const float *xp, const float4 *tp, int nch, float (&acc)[CPT][ARS_RQ][4])
{
  constexpr int RQ = ARS_RQ;
#pragma unroll
  for (int u = 0; u < CPT; u++)
#pragma unroll
    for (int r = 0; r < RQ; r++)
#pragma unroll
      for (int k = 0; k < 4; k++) acc[u][r][k] = 0.f;
#pragma unroll 2
  for (int ch = 0; ch < nch; ch++, xp += 4 * CB, tp += RQ) {
    float x[CPT][4];
    if (CPT == 4) {
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const float4 v = *(const float4 *) (xp + k * CB);
        x[0][k] = v.x; x[1 % CPT][k] = v.y; x[2 % CPT][k] = v.z; x[3 % CPT][k] = v.w;
      }
    } else if (CPT == 2) {
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const float2 v = *(const float2 *) (xp + k * CB);
        x[0][k] = v.x; x[CPT - 1][k] = v.y;
      }
    } else {
#pragma unroll
      for (int k = 0; k < 4; k++) x[0][k] = xp[k * CB];
    }
#pragma unroll
    for (int r = 0; r < RQ; r++) {
      const float4 t = tp[r];
#pragma unroll
      for (int u = 0; u < CPT; u++) {
        acc[u][r][0] = __fadd_rn (acc[u][r][0], __fmul_rn (x[u][0], t.x));
        acc[u][r][1] = __fadd_rn (acc[u][r][1], __fmul_rn (x[u][1], t.y));
        acc[u][r][2] = __fadd_rn (acc[u][r][2], __fmul_rn (x[u][2], t.z));
        acc[u][r][3] = __fadd_rn (acc[u][r][3], __fmul_rn (x[u][3], t.w));
      }
    }
  }
}

// the integer inner products' rounding: the S16 sum (wrapped to 32 bits) + 2^14, >> 15, saturated
// (audio-resampler-x86-sse2.c:48-54); the S32 sum (wrapped to 64 bits) + 2^30, >> 31, saturated
__device__ __forceinline__ int ars_round_s16 (unsigned sum) { return min (max ((int) (sum + (1u << 14)) >> 15, -32768), 32767); }
__device__ __forceinline__ int ars_round_s32 (unsigned long long sum)
{
  const long long v = ((long long) sum + (1 << 30)) >> 31;
  return (int) (v < -2147483648LL ? -2147483648LL : (v > 2147483647LL ? 2147483647LL : v));
}

__global__ void __launch_bounds__ (ARS_THREADS)
ars_full_kernel (const ArsLaunch L)
{
  extern __shared__ __align__ (16) float rows[];                // [no][row_pitch]
  __shared__ long long s_idx[64];
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync (0xffffffffu, (int) (threadIdx.x >> 5), 0);
  const long long o0 = (long long) blockIdx.x * L.no;
  const int n_out = (int) min ((long long) L.no, L.out_frames - o0);

  // stage this CTA's tap rows, each shifted by (window start & 3) and zero padded
  for (int j = warp; j < n_out; j += ARS_THREADS / 32) {
    long long idx; int phase;
    ars_position (L, o0 + j, idx, phase);
    if (lane == 0) s_idx[j] = idx;
    const int delta = (int) (idx & 3);
    const float *src = L.phases + (size_t) phase * L.n_taps;
    float *dst = rows + (size_t) j * L.row_pitch;
    for (int m = lane; m < L.row_pitch; m += 32) {
      const int k = m - delta;
      dst[m] = (k >= 0 && k < L.n_taps) ? __ldg (src + k) : 0.f;
    }
  }
  __syncthreads ();

  const int cg = warp % L.wcn, og = warp / L.wcn, nog = (ARS_THREADS / 32) / L.wcn;
  const int c = (blockIdx.y * L.wcn + cg) * 32 + lane;
  const bool c_ok = c < L.channels;
  const int cc = c_ok ? c : L.channels - 1;
  for (int q = og * ARS_RQ; q < n_out; q += nog * ARS_RQ) {
    long long idx[ARS_RQ];
    float acc[ARS_RQ][4];
#pragma unroll
    for (int r = 0; r < ARS_RQ; r++) {
      idx[r] = s_idx[min (q + r, n_out - 1)];
#pragma unroll
      for (int j = 0; j < 4; j++) acc[r][j] = 0.f;
    }
    const long long s_begin = idx[0] & ~3LL;
    const long long s_end = idx[ARS_RQ - 1] + L.n_taps;
    for (long long s4 = s_begin; s4 < s_end; s4 += 4) {
      float x[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        // two loads rather than ars_frame_row's pointer: selecting the row first costs this kernel two registers
        const long long f = s4 + j;
        float v = 0.f;
        if (f < L.hist_frames) v = __ldg (L.hist + f * L.channels + cc);
        else if (f < L.avail && L.in) v = __ldg (L.in + (f - L.hist_frames) * L.channels + cc);
        x[j] = v;
      }
#pragma unroll
      for (int r = 0; r < ARS_RQ; r++) {
        const long long k0 = s4 - idx[r];                        // tap index of x[0]
        if (k0 <= -4 || k0 >= L.n_taps) continue;                // warp-uniform
        const int m0 = (int) (s4 - (idx[r] & ~3LL));             // aligned column in the shifted row
        const float4 t = *(const float4 *) (rows + (size_t) min (q + r, n_out - 1) * L.row_pitch + m0);
        if (k0 >= 0 && k0 + 3 < L.n_taps) {
          acc[r][0] = __fadd_rn (acc[r][0], __fmul_rn (x[0], t.x));
          acc[r][1] = __fadd_rn (acc[r][1], __fmul_rn (x[1], t.y));
          acc[r][2] = __fadd_rn (acc[r][2], __fmul_rn (x[2], t.z));
          acc[r][3] = __fadd_rn (acc[r][3], __fmul_rn (x[3], t.w));
        } else {                                                 // window edge: skip taps outside [0, n_taps)
          if (k0 + 0 >= 0 && k0 + 0 < L.n_taps) acc[r][0] = __fadd_rn (acc[r][0], __fmul_rn (x[0], t.x));
          if (k0 + 1 >= 0 && k0 + 1 < L.n_taps) acc[r][1] = __fadd_rn (acc[r][1], __fmul_rn (x[1], t.y));
          if (k0 + 2 >= 0 && k0 + 2 < L.n_taps) acc[r][2] = __fadd_rn (acc[r][2], __fmul_rn (x[2], t.z));
          if (k0 + 3 >= 0 && k0 + 3 < L.n_taps) acc[r][3] = __fadd_rn (acc[r][3], __fmul_rn (x[3], t.w));
        }
      }
    }
#pragma unroll
    for (int r = 0; r < ARS_RQ; r++) {
      if (q + r < n_out && c_ok) L.out[(size_t) (o0 + q + r) * L.channels + c] = ars_lane_sum (acc[r]);
    }
  }
}

// Fast path: the CTA's whole input window is staged in shared memory once (frames x channel
// block) and the taps of each group of RQ consecutive outputs are laid out chunk-major
// ([chunk][output] float4, zero outside each output's window), so the inner loop is branch free:
// per 4-frame chunk 4 LDS (inputs, immediate offsets) + RQ LDS.128 (broadcast taps) + 4*RQ FMUL
// + 4*RQ FADD and two pointer bumps.  A zero tap contributes x*0 = +-0, which leaves the
// partial sums unchanged for finite input (the sums start at +0 and can never become -0).
struct ArsTile {
  int win;                       // staged frames per CTA (multiple of 4)
  int nch;                       // chunks per output group (upper bound, fixed stride of the tap table)
  // chunk-major taps of every possible 4-output group, laid out on the host once per plan (F32 only):
  // qtab[((a * out_step + phase) * nch + chunk) * RQ + r], a = (first window sample of the group) mod 4, phase = its filter
  // phase.  A CTA copies the rows of its groups instead of gathering taps one by one with bounds tests.
  const float4 *qtab;
};

// win and nch of a CTA that produces `no` consecutive outputs (qtab left null); nch does not depend on `no`
static ArsTile ars_tile_geometry (const ArsPlan & p, int no)
{
  ArsTile t = ArsTile ();
  // frames spanned by `no` outputs: ceil (no * in_step / out_step) + alignment + taps
  const long long span = ((long long) no * p.in_step + p.out_step - 1) / p.out_step + 8 + p.n_taps;
  t.win = (int) ((span + 3) & ~3LL);
  const long long spread = ((long long) (ARS_RQ - 1) * p.in_step + p.out_step - 1) / p.out_step + 1;
  t.nch = (int) ((spread + p.n_taps + 3 + 3) / 4 + 1);
  return t;
}

// shared memory of a tile kernel CTA: the chunk-major taps of its no / RQ output groups, then its window of cb channels
static size_t ars_tile_smem (const ArsTile & t, int no, int cb, int sample_bytes)
{
  return (size_t) (no / ARS_RQ) * t.nch * ARS_RQ * 4 * sizeof (float) + (size_t) t.win * cb * sample_bytes;
}

// host side of the layout above; phases = [phase][n_taps] taps of type Tap, stored as Wide (4 bytes: F32 taps as they
// are, the S16 resampler's int16 taps widened to int32); nch from ars_tile_geometry
template <typename Tap, typename Wide>
static void ars_build_qtab (const ArsPlan & p, const Tap *phases, int nch, std::vector<float> * out)
{
  static_assert (sizeof (Wide) == sizeof (float), "the table is uploaded as floats");
  const int RQ = 4;
  out->assign ((size_t) 4 * p.out_step * nch * RQ * 4, 0.f);
  Wide *o = (Wide *) out->data ();
  for (int a = 0; a < 4; a++)
    for (int ph = 0; ph < p.out_step; ph++)
      for (int r = 0; r < RQ; r++) {
        const long long t = (long long) ph + (long long) r * p.samp_frac;
        const int delta = (int) ((long long) r * p.samp_inc + t / p.out_step), phase = (int) (t % p.out_step);
        const Tap *src = phases + (size_t) phase * p.n_taps;
        for (int chunk = 0; chunk < nch; chunk++) {
          Wide *dst = o + ((((size_t) a * p.out_step + ph) * nch + chunk) * RQ + r) * 4;
          for (int k = 0; k < 4; k++) {
            const int tap = 4 * chunk + k - (a + delta);
            dst[k] = (tap >= 0 && tap < p.n_taps) ? (Wide) src[tap] : (Wide) 0;
          }
        }
      }
}

template <int CB, int CPT>
__global__ void __launch_bounds__ (ARS_THREADS)
ars_tile_kernel (const ArsLaunch L, const ArsTile Tl)
{
  extern __shared__ __align__ (16) float sm[];
  constexpr int RQ = ARS_RQ;
  const int nq_max = L.no / RQ;
  float4 *qt = (float4 *) sm;                                    // [nq][nch][RQ]
  float *xin = sm + (size_t) nq_max * Tl.nch * RQ * 4;           // [win][CB]
  __shared__ int s_rel[64], s_phase[64];
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync (0xffffffffu, (int) (threadIdx.x >> 5), 0);
  const long long o0 = (long long) blockIdx.x * L.no;
  const int n_out = (int) min ((long long) L.no, L.out_frames - o0);
  const int nq = (n_out + RQ - 1) / RQ;
  long long f0; int ph0;
  ars_position (L, o0, f0, ph0);
  f0 &= ~3LL;                                                    // chunk aligned window origin

  if (threadIdx.x < L.no) {
    long long idx; int phase;
    ars_position (L, o0 + min ((int) threadIdx.x, n_out - 1), idx, phase);
    s_rel[threadIdx.x] = (int) (idx - f0);
    s_phase[threadIdx.x] = phase;
  }
  // stage the input window row by row (one warp per frame, coalesced)
  const int c_base = blockIdx.y * CB;
  // CB == 128 with whole, 16-byte aligned channel blocks: a lane moves 4 channels of a frame (LDG.128 -> STS.128)
  const bool vec = CB == 128 && (L.channels & 3) == 0 && c_base + CB <= L.channels &&
      ((((uintptr_t) L.hist) | ((uintptr_t) L.in)) & 15) == 0;
  for (int fr = warp; fr < Tl.win; fr += ARS_THREADS / 32) {
    const float *src = ars_frame_row<float> (L, f0 + fr);
    if (vec) {
      *(float4 *) (xin + fr * CB + 4 * lane) = src ? __ldg ((const float4 *) (src + c_base) + lane) : make_float4 (0.f, 0.f, 0.f, 0.f);
    } else {
#pragma unroll
      for (int c = lane; c < CB; c += 32)
        xin[fr * CB + c] = (src && c_base + c < L.channels) ? __ldg (src + c_base + c) : 0.f;
    }
  }
  __syncthreads ();
  // chunk-major tap table: the rows of this CTA's output groups, copied from the plan's pre-laid table
  {
    const int row = Tl.nch * RQ;                                  // float4 per group
    const int e = threadIdx.x & 127, qq = threadIdx.x >> 7;       // two groups per pass, up to 128 float4 each
    for (int q = qq; q < nq; q += ARS_THREADS / 128) {
      const float4 *src = Tl.qtab + ((size_t) (s_rel[q * RQ] & 3) * L.out_step + s_phase[q * RQ]) * row;
      for (int i = e; i < row; i += 128) qt[q * row + i] = __ldg (src + i);
    }
  }
  __syncthreads ();

  // a thread owns CPT adjacent channels x RQ consecutive outputs: every broadcast tap quad (LDS.128)
  // then feeds CPT channels, which halves the shared-memory traffic per multiply for CPT = 2
  constexpr int WCN = CB / (32 * CPT);
  const int cg = warp % WCN, og = warp / WCN;
  constexpr int NOG = (ARS_THREADS / 32) / WCN;
  const int cl = (cg * 32 + lane) * CPT, c = c_base + cl;
  for (int q = og; q < nq; q += NOG) {
    const int s_min = s_rel[q * RQ] & ~3;
    const int s_max = (s_rel[min (q * RQ + RQ - 1, n_out - 1)] + L.n_taps + 3) & ~3;
    const int nch = (s_max - s_min) >> 2;
    const float *xp = xin + s_min * CB + cl;
    const float4 *tp = qt + (size_t) q * Tl.nch * RQ;
    float acc[CPT][RQ][4];
    ars_group_f32<CPT, CB> (xp, tp, nch, acc);
#pragma unroll
    for (int r = 0; r < RQ; r++) {
#pragma unroll
      for (int u = 0; u < CPT; u++) {
        if (q * RQ + r < n_out && c + u < L.channels)
          L.out[(size_t) (o0 + q * RQ + r) * L.channels + c + u] = ars_lane_sum (acc[u][r]);
      }
    }
  }
}

// ---- ars_pipe_kernel: the tile kernel as a persistent, double-buffered pipeline ------------------------------------------
// In ars_tile_kernel on the C5 shape the prologue (window and tap rows travelling from L2 to shared memory) stalls far more
// than its share of the instructions - two CTAs per SM cannot hide it.
// Here one CTA per SM (16 warps) walks its tiles (64 outputs x 128 channels) with TWO staging buffers: while the warps
// multiply tile k, cp.async fills the window and the tap rows of tile k+1 (zero fill for silence / missing frames through
// the src-size operand).  With registers no longer shared between CTAs a thread owns 4 adjacent channels x 4 outputs:
// one LDS.128 of samples and one broadcast LDS.128 of taps feed 32 FMUL + 32 FADD.  Arithmetic and its order are those of
// ars_tile_kernel (four partial sums by tap index mod 4, (l0 + l2) + (l1 + l3), no FMA): bit-identical output.
constexpr int ARS_PIPE_THREADS = 512, ARS_PIPE_NO = 64, ARS_PIPE_CB = 128;

// sign-extending byte permute: the 16-bit sample in the low (0x9910) or high (0xbb32) half of a word as an int
__device__ __forceinline__ int prmt_s16 (unsigned v, unsigned sel)
{
#ifdef B200_CUDA_EMU
  return sel == 0x9910u ? (int) (short) (v & 0xffffu) : (int) (short) (v >> 16);
#else
  int d;
  asm ("prmt.b32 %0, %1, 0, %2;" : "=r" (d) : "r" (v), "r" (sel));
  return d;
#endif
}

// What the pipelines do per sample format: the staged Sample type (which sets the stage layout and the copy sizes), the
// Tap vector of one chunk of the tap rows, and group (): a warp's 4-output group for its lane's 4 adjacent channels c ..
// c + 3 - xp, tp and nch as for ars_group_f32; outputs o0 + q0 .. o0 + q0 + 3 of the stream, those below the tile's n_out
// stored.
struct ArsPipeF32 {
  typedef float Sample;
  typedef float4 Tap;
  static __device__ __forceinline__ void group (const ArsLaunch & L, const float *xp, const float4 *tp, int nch, long long o0, int q0, int c, int n_out)
  {
    float acc[4][ARS_RQ][4];
    ars_group_f32<4, ARS_PIPE_CB> (xp, tp, nch, acc);
    float *op = L.out + (size_t) (o0 + q0) * L.channels + c;
#pragma unroll
    for (int r = 0; r < ARS_RQ; r++) {
      if (q0 + r < n_out) {
        float4 o;
        o.x = ars_lane_sum (acc[0][r]); o.y = ars_lane_sum (acc[1][r]); o.z = ars_lane_sum (acc[2][r]); o.w = ars_lane_sum (acc[3][r]);
        *(float4 *) (op + (size_t) r * L.channels) = o;
      }
    }
  }
};

// The window travels as raw 16-bit samples, the tap rows as 32-bit ints in the F32 chunk-major layout: per frame position
// one LDS.64 of samples (4 sign-extending PRMT) and per output one broadcast LDS.128 of taps feed 16 IMAD.  Integer sums
// wrap in 32 bits like the SSE2 pmaddwd path (inner_product_gint16_full_1_sse2, audio-resampler-x86-sse2.c:29-56): no lane
// structure to keep, one accumulator per (channel, output).
struct ArsPipeS16 {
  typedef short Sample;
  typedef int4 Tap;
  static __device__ __forceinline__ void group (const ArsLaunch & L, const short *xp, const int4 *tp, int nch, long long o0, int q0, int c, int n_out)
  {
    constexpr int RQ = ARS_RQ, CB = ARS_PIPE_CB;
    unsigned acc[4][RQ];
#pragma unroll
    for (int u = 0; u < 4; u++)
#pragma unroll
      for (int r = 0; r < RQ; r++) acc[u][r] = 0u;
#pragma unroll 2
    for (int ch = 0; ch < nch; ch++, xp += 4 * CB, tp += RQ) {
      int x[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; kk++) {
        const uint2 v = *(const uint2 *) (xp + kk * CB);           // 4 adjacent channels of one frame, 16 bits each
        x[0][kk] = prmt_s16 (v.x, 0x9910u); x[1][kk] = prmt_s16 (v.x, 0xbb32u);
        x[2][kk] = prmt_s16 (v.y, 0x9910u); x[3][kk] = prmt_s16 (v.y, 0xbb32u);
      }
#pragma unroll
      for (int r = 0; r < RQ; r++) {
        const int4 tq = tp[r];
#pragma unroll
        for (int u = 0; u < 4; u++)
          acc[u][r] += (unsigned) (x[u][0] * tq.x) + (unsigned) (x[u][1] * tq.y) + (unsigned) (x[u][2] * tq.z) + (unsigned) (x[u][3] * tq.w);
      }
    }
    short *op = (short *) L.out + (size_t) (o0 + q0) * L.channels + c;
#pragma unroll
    for (int r = 0; r < RQ; r++) {
      if (q0 + r < n_out) {
        const int v0 = ars_round_s16 (acc[0][r]), v1 = ars_round_s16 (acc[1][r]);
        const int v2 = ars_round_s16 (acc[2][r]), v3 = ars_round_s16 (acc[3][r]);
        uint2 o;
        o.x = ((unsigned) v0 & 0xffffu) | ((unsigned) v1 << 16);
        o.y = ((unsigned) v2 & 0xffffu) | ((unsigned) v3 << 16);
        *(uint2 *) (op + (size_t) r * L.channels) = o;
      }
    }
  }
};

__device__ __forceinline__ void ars_cp16 (void *dst_smem, const void *src, bool real)
{
#ifndef B200_CUDA_EMU
  const unsigned d = (unsigned) __cvta_generic_to_shared (dst_smem);
  const int bytes = real ? 16 : 0;                                // src-size 0: the 16 bytes are written as zeros
  asm volatile ("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r" (d), "l" (src), "r" (bytes) : "memory");
#else
  if (real) *(float4 *) dst_smem = *(const float4 *) src; else *(float4 *) dst_smem = make_float4 (0.f, 0.f, 0.f, 0.f);
#endif
}

__global__ void __launch_bounds__ (ARS_PIPE_THREADS, 1)
ars_pipe_kernel_v1 (const ArsLaunch L, const ArsTile Tl, int n_fb, int n_cb)
{
  extern __shared__ __align__ (16) float sm[];
  constexpr int RQ = ARS_RQ, NO = ARS_PIPE_NO, CB = ARS_PIPE_CB, NQ = NO / RQ;
  const int row = Tl.nch * RQ;                                    // float4 per output group in the tap table
  const size_t qt_floats = (size_t) NQ * row * 4, xin_floats = (size_t) Tl.win * CB;
  float *base[2] = {sm, sm + qt_floats + xin_floats};
  __shared__ int s_rel[3][NO], s_phase[3][NO];                    // positions run two tiles ahead, off the critical path
  __shared__ long long s_f0[3];
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync (0xffffffffu, (int) (threadIdx.x >> 5), 0);
  const int n_tiles = n_fb * n_cb;

  auto positions = [&] (int t, int b) {                           // threads < NO: where tile t's outputs sit in the stream (b: slot of 3)
    if (threadIdx.x < NO) {
      const long long o0 = (long long) (t / n_cb) * NO;
      const int n_out = (int) min ((long long) NO, L.out_frames - o0);
      long long f0; int ph0;
      ars_position (L, o0, f0, ph0);
      f0 &= ~3LL;
      long long idx; int phase;
      ars_position (L, o0 + min ((int) threadIdx.x, n_out - 1), idx, phase);
      s_rel[b][threadIdx.x] = (int) (idx - f0);
      s_phase[b][threadIdx.x] = phase;
      if (threadIdx.x == 0) s_f0[b] = f0;
    }
  };
  auto prefetch = [&] (int t, int b, int ps) {                    // all threads: cp.async of tile t into buffer b; ps: its position slot
    float4 *qt = (float4 *) base[b];
    float *xin = base[b] + qt_floats;
    const long long f0 = s_f0[ps];
    const int c_base = (t % n_cb) * CB;
    for (int fr = warp; fr < Tl.win; fr += ARS_PIPE_THREADS / 32) {
      const float *src = ars_frame_row<float> (L, f0 + fr);
      ars_cp16 (xin + fr * CB + 4 * lane, src ? (const void *) (src + c_base + 4 * lane) : (const void *) Tl.qtab, src != nullptr);
    }
    const int e = threadIdx.x & 127, qq = threadIdx.x >> 7;
    for (int q = qq; q < NQ; q += ARS_PIPE_THREADS / 128) {
      const float4 *src = Tl.qtab + ((size_t) (s_rel[ps][q * RQ] & 3) * L.out_step + s_phase[ps][q * RQ]) * row;
      for (int i = e; i < row; i += 128) ars_cp16 (qt + q * row + i, src + i, true);
    }
#ifndef B200_CUDA_EMU
    asm volatile ("cp.async.commit_group;" ::: "memory");
#endif
  };

  int t = blockIdx.x, b = 0, ps = 0;                              // ps: position slot of tile t (k mod 3)
  if (t < n_tiles) positions (t, 0);
  if (t + (int) gridDim.x < n_tiles) positions (t + gridDim.x, 1);
  __syncthreads ();
  if (t < n_tiles) prefetch (t, 0, 0);
  for (; t < n_tiles; t += gridDim.x, b ^= 1, ps = (ps + 1) % 3) {
    const int tn = t + gridDim.x, tnn = tn + gridDim.x;
#ifndef B200_CUDA_EMU
    asm volatile ("cp.async.wait_group 0;" ::: "memory");
#endif
    __syncthreads ();                                             // tile t staged; positions of tile t+1 visible (written an iteration ago)
    if (tn < n_tiles) prefetch (tn, b ^ 1, (ps + 1) % 3);
    if (tnn < n_tiles) positions (tnn, (ps + 2) % 3);             // overlaps this tile's arithmetic

    const float4 *qt = (const float4 *) base[b];
    const float *xin = base[b] + qt_floats;
    const long long o0 = (long long) (t / n_cb) * NO;
    const int n_out = (int) min ((long long) NO, L.out_frames - o0);
    const int nq = (n_out + RQ - 1) / RQ;
    const int c = (t % n_cb) * CB + 4 * lane;
    for (int q = warp; q < nq; q += ARS_PIPE_THREADS / 32) {
      const int s_min = s_rel[ps][q * RQ] & ~3;
      const int s_max = (s_rel[ps][min (q * RQ + RQ - 1, n_out - 1)] + L.n_taps + 3) & ~3;
      float acc[4][RQ][4];
      ars_group_f32<4, CB> (xin + s_min * CB + 4 * lane, qt + (size_t) q * row, (s_max - s_min) >> 2, acc);
#pragma unroll
      for (int r = 0; r < RQ; r++) {
        if (q * RQ + r < n_out) {
          float4 o;
          o.x = ars_lane_sum (acc[0][r]); o.y = ars_lane_sum (acc[1][r]); o.z = ars_lane_sum (acc[2][r]); o.w = ars_lane_sum (acc[3][r]);
          *(float4 *) (L.out + (size_t) (o0 + q * RQ + r) * L.channels + c) = o;
        }
      }
    }
    __syncthreads ();                                             // buffer b and its positions are free for tile t + 2
  }
}

// ---- ars_pipe_kernel (second form): bulk copies + mbarriers, no CTA-wide barrier in the steady state ----------------------
// In the cp.async form above a tenth of the instructions are cp.async issue + its address arithmetic (4800 16-byte copies
// per tile), the two __syncthreads per tile stall warps, and the stage pointers selected from a two-entry array made the inner loop's
// loads generic (LD.E.128) instead of LDS.128.  Here a window row (CB channels of one frame, 512 contiguous bytes) and a
// tap row (one 4-output group, nch * 64 bytes) each travel as ONE cp.async.bulk issued by one lane (166 per tile instead
// of 6080 cp.async), completion is counted by an mbarrier per stage (full[2]), and the stage is handed back through a
// second one (empty[2]) on which only the four producing warps ever wait - the other twelve go from tile to tile without
// meeting anybody.  Frames outside the stream (silence, start-up) are zero rows written by the producing lane itself.
// Arithmetic, its order and the staged layout are unchanged: bit-identical output.
struct alignas (16) ArsBar { unsigned long long w[2]; };         // w[0]: the mbarrier object (the emulated build uses all 16 bytes)
constexpr int ARS_PIPE_PROD = 4;                                  // producing warps (one per scheduler)

#ifdef B200_CUDA_EMU
}  // namespace b200 (reopened below)
#include <mutex>
#include <thread>
namespace b200 {
static std::mutex g_emu_bar_mu;
struct EmuBar { int count, pending, tx, phase; };
static_assert (sizeof (EmuBar) == sizeof (ArsBar), "emulated barrier must fit");
static inline void emu_bar_check (EmuBar *e) { if (e->pending == 0 && e->tx == 0) { e->phase ^= 1; e->pending = e->count; } }
#endif

__device__ __forceinline__ void ars_bar_init (ArsBar *bar, unsigned count)
{
#ifndef B200_CUDA_EMU
  asm volatile ("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r" ((unsigned) __cvta_generic_to_shared (bar)), "r" (count) : "memory");
#else
  EmuBar *e = (EmuBar *) bar; e->count = e->pending = (int) count; e->tx = 0; e->phase = 0;
#endif
}
__device__ __forceinline__ void ars_bar_arrive (ArsBar *bar)
{
#ifndef B200_CUDA_EMU
  asm volatile ("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r" ((unsigned) __cvta_generic_to_shared (bar)) : "memory");
#else
  std::lock_guard<std::mutex> l (g_emu_bar_mu); EmuBar *e = (EmuBar *) bar; e->pending--; emu_bar_check (e);
#endif
}
__device__ __forceinline__ void ars_bar_arrive_tx (ArsBar *bar, unsigned bytes)
{
#ifndef B200_CUDA_EMU
  asm volatile ("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r" ((unsigned) __cvta_generic_to_shared (bar)), "r" (bytes) : "memory");
#else
  std::lock_guard<std::mutex> l (g_emu_bar_mu); EmuBar *e = (EmuBar *) bar; e->tx += (int) bytes; e->pending--; emu_bar_check (e);
#endif
}
// waits until the phase of the given parity has completed; a lost arrival must fail loudly, not hang the device
__device__ __forceinline__ void ars_bar_wait (ArsBar *bar, unsigned parity)
{
#ifndef B200_CUDA_EMU
  const unsigned a = (unsigned) __cvta_generic_to_shared (bar);
  unsigned spins = 0;
  for (;;) {
    unsigned ok;
    asm volatile ("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r" (ok) : "r" (a), "r" (parity) : "memory");
    if (ok) break;
    if (++spins > (1u << 22)) __trap ();
  }
#else
  for (;;) {
    { std::lock_guard<std::mutex> l (g_emu_bar_mu); if ((unsigned) ((EmuBar *) bar)->phase != parity) break; }
    std::this_thread::yield ();
  }
#endif
}
// one contiguous global -> shared copy (16-byte aligned, size a multiple of 16) whose bytes count on `bar`
__device__ __forceinline__ void ars_bulk_g2s (void *dst_smem, const void *src, unsigned bytes, ArsBar *bar)
{
#ifndef B200_CUDA_EMU
  asm volatile ("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      :: "r" ((unsigned) __cvta_generic_to_shared (dst_smem)), "l" (src), "r" (bytes), "r" ((unsigned) __cvta_generic_to_shared (bar)) : "memory");
#else
  memcpy (dst_smem, src, bytes);
  std::lock_guard<std::mutex> l (g_emu_bar_mu); EmuBar *e = (EmuBar *) bar; e->tx -= (int) bytes; emu_bar_check (e);
#endif
}
// CUtensorMap as an opaque 128-byte kernel parameter (the emulated build has no driver types)
struct alignas (64) ArsTensorMap { unsigned long long opaque[16]; };
__device__ __forceinline__ void ars_tensor_g2s (void *dst_smem, const ArsTensorMap *tm, int c0, int c1, ArsBar *bar)
{
#ifndef B200_CUDA_EMU
  asm volatile ("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      :: "r" ((unsigned) __cvta_generic_to_shared (dst_smem)), "l" (tm), "r" (c0), "r" (c1),
         "r" ((unsigned) __cvta_generic_to_shared (bar)) : "memory");
#else
  (void) dst_smem; (void) tm; (void) c0; (void) c1; (void) bar;   // never taken: the emulated launch passes use_tm = 0
#endif
}
__device__ __forceinline__ void ars_warp_sync ()
{
#ifndef B200_CUDA_EMU
  __syncwarp ();
#else
  (void) __shfl_sync (0xffffffffu, 0u, 0);                        // the emulated shuffle is a warp barrier
#endif
}

// The pipeline of both sample formats; S (ArsPipeF32, ArsPipeS16) gives the staged sample type and the arithmetic.  A
// stage = the tap rows (NQ groups x nch chunks of 4-tap vectors) + the window (win frames x CB samples).
template <class S>
__device__ __forceinline__ void ars_pipe_body (const ArsLaunch & L, const ArsTile & Tl, int n_fb, int n_cb, const ArsTensorMap *tm_in, int use_tm)
{
  typedef typename S::Sample Sample;
  extern __shared__ __align__ (128) float smp[];
  constexpr int RQ = ARS_RQ, NO = ARS_PIPE_NO, CB = ARS_PIPE_CB, NQ = NO / RQ, NW = ARS_PIPE_THREADS / 32;
  constexpr unsigned SB = sizeof (Sample);
  const int row = Tl.nch * RQ;                                    // tap vectors per output group in the tap table
  const unsigned qt_floats = (unsigned) NQ * row * 4, stage_floats = qt_floats + (unsigned) Tl.win * CB / (4 / SB);
  __shared__ ArsBar s_full[2], s_empty[2];
  __shared__ int s_rel[2][NO];
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync (0xffffffffu, (int) (threadIdx.x >> 5), 0);
  const int n_tiles = n_fb * n_cb;
  if (threadIdx.x == 0) {
    ars_bar_init (&s_full[0], ARS_PIPE_PROD); ars_bar_init (&s_full[1], ARS_PIPE_PROD);
    ars_bar_init (&s_empty[0], NW); ars_bar_init (&s_empty[1], NW);
#ifndef B200_CUDA_EMU
    asm volatile ("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
  }
  __syncthreads ();

  // producing warps: positions of tile t's outputs, one bulk copy per tap row and per window row into stage b
  auto produce = [&] (int t, int b) {
    float *stage = smp + (size_t) b * stage_floats;
    float4 *qt = (float4 *) stage;
    float *xin = stage + qt_floats;
    const int fb = t / n_cb, c_base = (t - fb * n_cb) * CB;
    const long long o0 = (long long) fb * NO;
    const int n_out = (int) min ((long long) NO, L.out_frames - o0);
    long long f0; int ph0;
    ars_position (L, o0, f0, ph0);
    f0 &= ~3LL;
#ifndef B200_CUDA_EMU
    asm volatile ("fence.proxy.async.shared::cta;" ::: "memory");  // zero rows written two tiles ago vs this tile's bulk writes
#endif
    unsigned tx = 0;
    if (lane < NO / ARS_PIPE_PROD) {
      const int j = warp * (NO / ARS_PIPE_PROD) + lane;
      long long idx; int phase;
      ars_position (L, o0 + min (j, n_out - 1), idx, phase);
      const int rel = (int) (idx - f0);
      s_rel[b][j] = rel;
      if ((j & (RQ - 1)) == 0) {
        const float4 *src = Tl.qtab + ((size_t) (rel & 3) * L.out_step + phase) * row;
        ars_bulk_g2s (qt + (size_t) (j / RQ) * row, src, (unsigned) row * 16u, &s_full[b]);
        tx += (unsigned) row * 16u;
      }
    }
    // a window that lies in the caller's input (every tile but the first few) is ONE tensor copy: box = CB channels x win
    // frames, rows past the end of the input arrive as zeros (out-of-bounds fill) like the missing frames of the row path.
    // (Divergent lanes issuing a bulk copy each are serialised through the uniform datapath: the row path below costs the
    // producing warps ~40 copies each and makes them the tile's stragglers.)
    const bool tensor = use_tm && f0 >= L.hist_frames;
    if (tensor) {
      if (warp == 0 && lane == 0) {
        ars_tensor_g2s (xin, tm_in, c_base, (int) (f0 - L.hist_frames), &s_full[b]);
        tx += (unsigned) Tl.win * CB * SB;
      }
    } else
    for (int fr = warp + ARS_PIPE_PROD * lane; fr < Tl.win; fr += 32 * ARS_PIPE_PROD) {
      const Sample *src = ars_frame_row<Sample> (L, f0 + fr);
      float *dst = xin + (size_t) fr * (CB * SB / 4);
      if (src) { ars_bulk_g2s (dst, src + c_base, CB * SB, &s_full[b]); tx += CB * SB; }
      else {
#pragma unroll 4
        for (int i = 0; i < (int) (CB * SB / 16); i++) ((float4 *) dst)[i] = make_float4 (0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) tx += __shfl_down_sync (0xffffffffu, tx, d);
    ars_warp_sync ();                                             // the lanes' s_rel entries and zero rows before lane 0's release
    if (lane == 0) ars_bar_arrive_tx (&s_full[b], tx);
  };

  int t = blockIdx.x, k = 0;
  if (warp < ARS_PIPE_PROD && t < n_tiles) produce (t, 0);
  for (; t < n_tiles; t += gridDim.x, k++) {
    const int b = k & 1, tn = t + gridDim.x;
    if (warp < ARS_PIPE_PROD && tn < n_tiles) {
      if (k >= 1) ars_bar_wait (&s_empty[b ^ 1], (unsigned) ((k - 1) >> 1) & 1u);   // every warp is done with tile k - 1
      produce (tn, b ^ 1);
    }
    ars_bar_wait (&s_full[b], (unsigned) (k >> 1) & 1u);

    const typename S::Tap *qt = (const typename S::Tap *) (smp + (size_t) b * stage_floats);
    const Sample *xin = (const Sample *) (smp + (size_t) b * stage_floats + qt_floats);
    const int fb = t / n_cb;
    const long long o0 = (long long) fb * NO;
    const int n_out = (int) min ((long long) NO, L.out_frames - o0);
    const int nq = (n_out + RQ - 1) / RQ;
    const int c = (t - fb * n_cb) * CB + 4 * lane;
    for (int q = warp; q < nq; q += NW) {
      const int s_min = s_rel[b][q * RQ] & ~3;
      const int s_max = (s_rel[b][min (q * RQ + RQ - 1, n_out - 1)] + L.n_taps + 3) & ~3;
      S::group (L, xin + s_min * CB + 4 * lane, qt + (size_t) q * row, (s_max - s_min) >> 2, o0, q * RQ, c, n_out);
    }
    ars_warp_sync ();
    if (lane == 0) ars_bar_arrive (&s_empty[b]);                  // this warp no longer reads stage b
  }
}

__global__ void __launch_bounds__ (ARS_PIPE_THREADS, 1)
ars_pipe_kernel (const ArsLaunch L, const ArsTile Tl, int n_fb, int n_cb, const __grid_constant__ ArsTensorMap tm_in, int use_tm)
{
  ars_pipe_body<ArsPipeF32> (L, Tl, n_fb, n_cb, &tm_in, use_tm);
}

// ---- ars_pipe_kernel_s16: the same pipeline for S16 streams ----------------------------------------------------------------
// The window travels as raw 16-bit samples (one tensor copy of half the bytes), the tap rows as 32-bit ints (ars_build_qtab
// <int16_t, int32_t>); the IMADs (half rate) bound it exactly where FMUL + FADD bound the F32 kernel.  Sums wrap in 32 bits,
// + 2^14, >> 15, saturate: byte-identical to ars_tile_kernel_s16.
__global__ void __launch_bounds__ (ARS_PIPE_THREADS, 1)
ars_pipe_kernel_s16 (const ArsLaunch L, const ArsTile Tl, int n_fb, int n_cb, const __grid_constant__ ArsTensorMap tm_in, int use_tm)
{
  ars_pipe_body<ArsPipeS16> (L, Tl, n_fb, n_cb, &tm_in, use_tm);
}

// S16 samples through the tile kernel's tiling: the window is staged widened to 32 bits, taps likewise; the sums are
// integers (wrapping 32 bit like the SSE2 pmaddwd path), so no lane structure has to be kept —
// inner_product_gint16_full_1_sse2 (audio-resampler-x86-sse2.c:29-56): sum, + 2^14, >> 15, saturate.
template <int CB>
__global__ void __launch_bounds__ (ARS_THREADS)
ars_tile_kernel_s16 (const ArsLaunch L, const ArsTile Tl)
{
  extern __shared__ __align__ (16) float sm[];
  constexpr int RQ = ARS_RQ, CPT = 2;
  const int nq_max = L.no / RQ;
  int4 *qt = (int4 *) sm;                                        // [nq][nch][RQ]
  int *xin = (int *) sm + (size_t) nq_max * Tl.nch * RQ * 4;      // [win][CB]
  __shared__ int s_rel[64], s_phase[64];
  const short *phases = (const short *) L.phases;
  short *out = (short *) L.out;
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync (0xffffffffu, (int) (threadIdx.x >> 5), 0);
  const long long o0 = (long long) blockIdx.x * L.no;
  const int n_out = (int) min ((long long) L.no, L.out_frames - o0);
  const int nq = (n_out + RQ - 1) / RQ;
  long long f0; int ph0;
  ars_position (L, o0, f0, ph0);
  f0 &= ~3LL;
  if (threadIdx.x < L.no) {
    long long idx; int phase;
    ars_position (L, o0 + min ((int) threadIdx.x, n_out - 1), idx, phase);
    s_rel[threadIdx.x] = (int) (idx - f0);
    s_phase[threadIdx.x] = phase;
  }
  const int c_base = blockIdx.y * CB;
  for (int fr = warp; fr < Tl.win; fr += ARS_THREADS / 32) {
    const short *src = ars_frame_row<short> (L, f0 + fr);
#pragma unroll
    for (int c = lane; c < CB; c += 32)
      xin[fr * CB + c] = (src && c_base + c < L.channels) ? (int) __ldg (src + c_base + c) : 0;
  }
  __syncthreads ();
  for (int i = threadIdx.x; i < nq * Tl.nch * RQ; i += ARS_THREADS) {
    const int r = i % RQ, chunk = (i / RQ) % Tl.nch, q = i / (RQ * Tl.nch);
    const int j = q * RQ + r;
    const int s_min = s_rel[q * RQ] & ~3;
    const int k0 = s_min + 4 * chunk - s_rel[j];
    const short *src = phases + (size_t) s_phase[j] * L.n_taps;
    int4 t;
    t.x = (k0 + 0 >= 0 && k0 + 0 < L.n_taps) ? (int) __ldg (src + k0 + 0) : 0;
    t.y = (k0 + 1 >= 0 && k0 + 1 < L.n_taps) ? (int) __ldg (src + k0 + 1) : 0;
    t.z = (k0 + 2 >= 0 && k0 + 2 < L.n_taps) ? (int) __ldg (src + k0 + 2) : 0;
    t.w = (k0 + 3 >= 0 && k0 + 3 < L.n_taps) ? (int) __ldg (src + k0 + 3) : 0;
    qt[i] = t;
  }
  __syncthreads ();

  constexpr int WCN = CB / (32 * CPT);
  const int cg = warp % WCN, og = warp / WCN;
  constexpr int NOG = (ARS_THREADS / 32) / WCN;
  const int cl = (cg * 32 + lane) * CPT, c = c_base + cl;
  for (int q = og; q < nq; q += NOG) {
    unsigned acc[CPT][RQ];
#pragma unroll
    for (int u = 0; u < CPT; u++)
#pragma unroll
      for (int r = 0; r < RQ; r++) acc[u][r] = 0u;
    const int s_min = s_rel[q * RQ] & ~3;
    const int s_max = (s_rel[min (q * RQ + RQ - 1, n_out - 1)] + L.n_taps + 3) & ~3;
    const int nch = (s_max - s_min) >> 2;
    const int *xp = xin + s_min * CB + cl;
    const int4 *tp = qt + (size_t) q * Tl.nch * RQ;
#pragma unroll 2
    for (int ch = 0; ch < nch; ch++, xp += 4 * CB, tp += RQ) {
      int x[CPT][4];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int2 v = *(const int2 *) (xp + k * CB);
        x[0][k] = v.x; x[1][k] = v.y;
      }
#pragma unroll
      for (int r = 0; r < RQ; r++) {
        const int4 t = tp[r];
#pragma unroll
        for (int u = 0; u < CPT; u++)
          acc[u][r] += (unsigned) (x[u][0] * t.x) + (unsigned) (x[u][1] * t.y) + (unsigned) (x[u][2] * t.z) + (unsigned) (x[u][3] * t.w);
      }
    }
#pragma unroll
    for (int r = 0; r < RQ; r++)
#pragma unroll
      for (int u = 0; u < CPT; u++)
        if (q * RQ + r < n_out && c + u < L.channels)
          out[(size_t) (o0 + q * RQ + r) * L.channels + c + u] = (short) ars_round_s16 (acc[u][r]);
  }
}

// Interpolated filter mode (audio-resampler.c:567-600 get_taps_gfloat_cubic +
// inner_product_gfloat_cubic_1_sse, audio-resampler-x86-sse.c:82-120): too many phases to cache, so
// every output takes four inner products against adjacent rows of the oversampled prototype and
// blends the four lane sums with the cubic coefficients of its own fractional position.
// Warp = one output frame x 32 channels; the prototype rows are warp-uniform LDG.128.
// Lane sums follow the tap index mod 4 as in the reference; (c0*f0 + c1*f1) + (c2*f2 + c3*f3)
// per lane, then (l0 + l2) + (l1 + l3).  No FMA anywhere.
// LIN: sinc-filter-interpolation=linear (get_taps_gfloat_linear + inner_product_gfloat_linear_1_sse,
// audio-resampler-x86-sse.c:48-74): two rows, blended per lane as (s0 - s1) * x + s1.
template <bool LIN>
__global__ void __launch_bounds__ (ARS_THREADS)
ars_interp_kernel (const ArsLaunch L, const float *__restrict__ table, int oversample)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long o = (long long) blockIdx.x * (ARS_THREADS / 32) + warp;
  if (o >= L.out_frames) return;
  const int c = blockIdx.y * 32 + lane;
  long long idx; int phase;
  ars_position (L, o, idx, phase);
  const long long pos = (long long) phase * oversample;
  const int offset = (oversample - 1) - (int) (pos / L.out_step), frac = (int) (pos % L.out_step);
  // make_coeff_gfloat_cubic (audio-resampler.c:360-373), evaluated in float like the reference
  const float x = __fdiv_rn (__int2float_rn (frac), __int2float_rn (L.out_step));
  const float x2 = __fmul_rn (x, x), x3 = __fmul_rn (x2, x);
  const float ic0 = __fmul_rn (0.16667f, __fsub_rn (x3, x));
  const float ic1 = __fadd_rn (x, __fmul_rn (0.5f, __fsub_rn (x2, x3)));
  const float ic3 = __fsub_rn (__fadd_rn (__fmul_rn (-0.33333f, x), __fmul_rn (0.5f, x2)), __fmul_rn (0.16667f, x3));
  const float ic2 = __fsub_rn (__fsub_rn (__fsub_rn (1.0f, ic0), ic1), ic3);
  const float4 *row = (const float4 *) (table + (size_t) offset * L.n_taps);
  const int rstride = L.n_taps >> 2;
  constexpr int ROWS = LIN ? 2 : 4;
  float acc[4][4];
#pragma unroll
  for (int k = 0; k < 4; k++)
#pragma unroll
    for (int l = 0; l < 4; l++) acc[k][l] = 0.f;
  const bool live = c < L.channels;
  for (int i = 0; i < L.n_taps; i += 4) {
    float xs[4];
#pragma unroll
    for (int l = 0; l < 4; l++) {
      const long long f = idx + i + l;
      float v = 0.f;
      if (live) {
        if (f < L.hist_frames) v = __ldg (L.hist + f * L.channels + c);
        else if (L.in) v = __ldg (L.in + (f - L.hist_frames) * L.channels + c);
      }
      xs[l] = v;
    }
#pragma unroll
    for (int k = 0; k < ROWS; k++) {
      const float4 t = __ldg (row + k * rstride + (i >> 2));
      acc[k][0] = __fadd_rn (acc[k][0], __fmul_rn (xs[0], t.x));
      acc[k][1] = __fadd_rn (acc[k][1], __fmul_rn (xs[1], t.y));
      acc[k][2] = __fadd_rn (acc[k][2], __fmul_rn (xs[2], t.z));
      acc[k][3] = __fadd_rn (acc[k][3], __fmul_rn (xs[3], t.w));
    }
  }
  float t[4];
#pragma unroll
  for (int l = 0; l < 4; l++)
    if (LIN)                    // make_coeff_gfloat_linear (:333-340): ic[0] = x
      t[l] = __fadd_rn (__fmul_rn (__fsub_rn (acc[0][l], acc[1][l]), x), acc[1][l]);
    else
      t[l] = __fadd_rn (__fadd_rn (__fmul_rn (acc[0][l], ic0), __fmul_rn (acc[1][l], ic1)),
          __fadd_rn (__fmul_rn (acc[2][l], ic2), __fmul_rn (acc[3][l], ic3)));
  if (live)
    L.out[(size_t) o * L.channels + c] = ars_lane_sum (t);
}

// ------------------------------------------------------------------------------------------
// S16 / S32 / F64 samples (audio-resampler.c macros, audio-resampler-x86-sse2.c, -sse41.c — the
// implementations an x86 build of the reference selects).  Integer sums are exact, so only the
// rounding points matter; F64 keeps the SSE2 two-lane order (lanes by tap parity, mul then add).
// Warp = one output frame x 32 channels; taps / prototype rows are warp-uniform loads.
struct ArsLaunchX {
  const void *hist, *in;
  void *out;
  const void *table;             // FULL: [n_phases][n_taps] taps; interpolated: [oversample + 4 (2: linear)][n_taps] prototype
  long long hist_frames, avail, out_frames;
  int channels, n_taps, out_step, samp_inc, samp_frac, samp_index, samp_phase;
  int full, oversample;
};
// make_coeff_gint16_linear / _gint32_linear (audio-resampler.c:325-332): ic[0] = x, ic[1] = 2^prec - 1 - x
__device__ __forceinline__ int linear_coeff_int (int frac, int denom, int prec)
{
  return (int) (((long long) frac << prec) / denom);
}

template <typename T>
__device__ __forceinline__ T ars_sample (const ArsLaunchX & L, long long f, int c)
{
  if (f < L.hist_frames) return __ldg ((const T *) L.hist + f * L.channels + c);
  if (L.in) return __ldg ((const T *) L.in + (f - L.hist_frames) * L.channels + c);
  return (T) 0;
}

// ---- packed samples: unpack, quantize, pack (audio-format.c MAKE_ORC_PACK_UNPACK / MAKE_PACK_UNPACK :116-217, the ORC
// programs of gstaudiopack.orc, audio-quantize.c gst_audio_quantize_quantize_int_none_none :88-95)
__device__ __forceinline__ unsigned long long ars_read_bytes (const ArsIo & io, const unsigned char *p)
{
  unsigned long long x = 0;
  for (int b = 0; b < io.step; b++) x |= (unsigned long long) __ldg (p + b) << (8 * (io.big ? io.step - 1 - b : b));
  return x;
}
__device__ __forceinline__ void ars_write_bytes (const ArsIo & io, unsigned char *p, unsigned long long x)
{
  for (int b = 0; b < io.step; b++) p[b] = (unsigned char) (x >> (8 * (io.big ? io.step - 1 - b : b)));
}
// the _trunc unpackers: the sample's bits moved to the top of 32 (bits shifted past bit 31 are lost), the sign bit flipped
// for unsigned formats
__device__ __forceinline__ int ars_unpack_int (const ArsIo & io, const unsigned char *p)
{
  return (int) (((unsigned) ars_read_bytes (io, p) << io.shift) ^ io.sign);
}
// bit casts and the double -> float narrowing (round to nearest), also in the emulated build
#ifndef B200_CUDA_EMU
__device__ __forceinline__ float ars_f32_of (unsigned b) { return __uint_as_float (b); }
__device__ __forceinline__ unsigned ars_bits_f32 (float f) { return __float_as_uint (f); }
__device__ __forceinline__ double ars_f64_of (unsigned long long b) { return __longlong_as_double ((long long) b); }
__device__ __forceinline__ unsigned long long ars_bits_f64 (double d) { return (unsigned long long) __double_as_longlong (d); }
__device__ __forceinline__ float ars_narrow (double d) { return __double2float_rn (d); }
#else
inline float ars_f32_of (unsigned b) { float f; memcpy (&f, &b, 4); return f; }
inline unsigned ars_bits_f32 (float f) { unsigned b; memcpy (&b, &f, 4); return b; }
inline double ars_f64_of (unsigned long long b) { double d; memcpy (&d, &b, 8); return d; }
inline unsigned long long ars_bits_f64 (double d) { unsigned long long b; memcpy (&b, &d, 8); return b; }
inline float ars_narrow (double d) { return (float) d; }
#endif
// ORC_DENORMAL: convfd / convdf flush denormals to a signed zero
__device__ __forceinline__ unsigned ars_flush_f32 (unsigned b) { return (b & 0x7f800000u) ? b : (b & 0xff800000u); }
__device__ __forceinline__ unsigned long long ars_flush_f64 (unsigned long long b)
{
  return (b & 0x7ff0000000000000ull) ? b : (b & 0xfff0000000000000ull);
}
__device__ __forceinline__ double ars_unpack_f64 (const ArsIo & io, const unsigned char *p)
{
  const unsigned long long x = ars_read_bytes (io, p);
  if (io.kind == ARS_IO_F32) return (double) ars_f32_of (ars_flush_f32 ((unsigned) x));
  return ars_f64_of (x);
}
// audio_orc_int_bias: saturating add of half a step, then the bits below the depth cleared; the pack's shift back down
__device__ __forceinline__ void ars_pack_int (const ArsIo & io, unsigned char *p, int v)
{
  if (io.qshift) {
    const long long t = (long long) v + (1LL << (io.qshift - 1));
    v = (int) (t > 2147483647LL ? 2147483647LL : t) & ~((1 << io.qshift) - 1);
  }
  const unsigned u = (unsigned) v ^ io.sign;
  ars_write_bytes (io, p, io.arith ? (unsigned) ((int) u >> io.shift) : u >> io.shift);
}
__device__ __forceinline__ void ars_pack_f64 (const ArsIo & io, unsigned char *p, double v)
{
  if (io.kind == ARS_IO_F32) {
    const float f = ars_narrow (ars_f64_of (ars_flush_f64 (ars_bits_f64 (v))));
    ars_write_bytes (io, p, ars_flush_f32 (ars_bits_f32 (f)));
  } else
    ars_write_bytes (io, p, ars_bits_f64 (v));
}

// How a kernel body reads a stream sample and writes an output sample.  ArsPlainIo: the caller's buffers hold the
// resampler's own format.  ArsPackedIo: the caller's samples are unpacked on load and quantized and packed on store; the
// history always holds the resampler's format.
struct ArsPlainIo {
  template <typename T> __device__ __forceinline__ T load (const ArsLaunchX & L, long long f, int c) const { return ars_sample<T> (L, f, c); }
  template <typename T> __device__ __forceinline__ void store (const ArsLaunchX & L, size_t at, T v) const { ((T *) L.out)[at] = v; }
};
struct ArsPackedIo {
  ArsIo io;
  template <typename T> __device__ __forceinline__ T load (const ArsLaunchX & L, long long f, int c) const
  {
    if (f < L.hist_frames) return __ldg ((const T *) L.hist + f * L.channels + c);
    if (!L.in) return (T) 0;
    const unsigned char *p = (const unsigned char *) L.in + (size_t) ((f - L.hist_frames) * L.channels + c) * io.step;
    return sizeof (T) == 8 ? (T) ars_unpack_f64 (io, p) : (T) ars_unpack_int (io, p);
  }
  template <typename T> __device__ __forceinline__ void store (const ArsLaunchX & L, size_t at, T v) const
  {
    unsigned char *p = (unsigned char *) L.out + at * io.step;
    if (sizeof (T) == 8) ars_pack_f64 (io, p, (double) v);
    else ars_pack_int (io, p, (int) v);
  }
};


template <int FMT, bool LIN, class IO>
__device__ __forceinline__ void ars_direct_body (const ArsLaunchX & L, const IO & io)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long o = (long long) blockIdx.x * (ARS_THREADS / 32) + warp;
  if (o >= L.out_frames) return;
  const int c = blockIdx.y * 32 + lane;
  if (c >= L.channels) return;
  const long long t0 = (long long) L.samp_phase + o * L.samp_frac;
  const long long idx = (long long) L.samp_index + o * L.samp_inc + t0 / L.out_step;
  const int phase = (int) (t0 % L.out_step), n = L.n_taps;
  // interpolated mode: first of the four prototype rows and the fractional position (get_taps_<type>_cubic)
  const long long pos = (long long) phase * L.oversample;
  const int offset = (L.oversample - 1) - (int) (pos / L.out_step), frac = (int) (pos % L.out_step);
  const size_t row0 = L.full ? (size_t) phase * n : (size_t) offset * n;

  if (FMT == ARS_S16) {
    const short *tab = (const short *) L.table + row0;
    if (L.full) {                 // inner_product_gint16_full_1_sse2
      unsigned sum = 0;
      for (int i = 0; i < n; i++) sum += (unsigned) ((int) io.template load<short> (L, idx + i, c) * (int) __ldg (tab + i));
      io.template store<short> (L, (size_t) o * L.channels + c, (short) ars_round_s16 (sum));
    } else if (LIN) {             // inner_product_gint16_linear_1_sse2 (audio-resampler-x86-sse2.c:57-108): 32-bit lane l
      unsigned s[2][4];           // sums the tap pairs (2l, 2l+1) of every eight; each LANE is shifted and multiplied
#pragma unroll
      for (int k = 0; k < 2; k++)
#pragma unroll
        for (int l = 0; l < 4; l++) s[k][l] = 0;
      for (int i = 0; i < n; i += 8)
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const int x = io.template load<short> (L, idx + i + j, c);
          s[0][j >> 1] += (unsigned) (x * (int) __ldg (tab + i + j));
          s[1][j >> 1] += (unsigned) (x * (int) __ldg (tab + n + i + j));
        }
      const int x = linear_coeff_int (frac, L.out_step, 15), y = 32767 - x;
      unsigned acc = 0;
#pragma unroll
      for (int l = 0; l < 4; l++)
        acc += (unsigned) ((int) (short) ((int) s[0][l] >> 15) * x) + (unsigned) ((int) (short) ((int) s[1][l] >> 15) * y);
      io.template store<short> (L, (size_t) o * L.channels + c, (short) ars_round_s16 (acc));
    } else {                      // inner_product_gint16_cubic_1_sse2
      unsigned s0 = 0, s1 = 0, s2 = 0, s3 = 0;
      for (int i = 0; i < n; i++) {
        const int x = io.template load<short> (L, idx + i, c);
        s0 += (unsigned) (x * (int) __ldg (tab + i));
        s1 += (unsigned) (x * (int) __ldg (tab + n + i));
        s2 += (unsigned) (x * (int) __ldg (tab + 2 * n + i));
        s3 += (unsigned) (x * (int) __ldg (tab + 3 * n + i));
      }
      int ic[4];
      cubic_coeff_s16 (frac, L.out_step, ic);
      const unsigned acc = (unsigned) ((int) (short) ((int) s0 >> 15) * ic[0]) + (unsigned) ((int) (short) ((int) s1 >> 15) * ic[1]) +
          (unsigned) ((int) (short) ((int) s2 >> 15) * ic[2]) + (unsigned) ((int) (short) ((int) s3 >> 15) * ic[3]);
      io.template store<short> (L, (size_t) o * L.channels + c, (short) ars_round_s16 (acc));
    }
  } else if (FMT == ARS_S32) {
    const int *tab = (const int *) L.table + row0;
    if (L.full) {                 // inner_product_gint32_full_1_sse41
      unsigned long long sum = 0;
      for (int i = 0; i < n; i++) sum += (unsigned long long) ((long long) io.template load<int> (L, idx + i, c) * __ldg (tab + i));
      io.template store<int> (L, (size_t) o * L.channels + c, ars_round_s32 (sum));
    } else {                      // inner_product_gint32_cubic_1_sse41: each 64-bit LANE (even / odd taps) is
      unsigned long long s[4][2]; // shifted and multiplied before the lanes are added; _linear_1_sse41 (:70-112) is the same
      constexpr int ROWS = LIN ? 2 : 4;   // arithmetic over two rows
#pragma unroll
      for (int k = 0; k < 4; k++) s[k][0] = s[k][1] = 0;
      for (int i = 0; i < n; i += 2) {
        const long long x0 = io.template load<int> (L, idx + i, c), x1 = io.template load<int> (L, idx + i + 1, c);
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
          s[k][0] += (unsigned long long) (x0 * __ldg (tab + k * n + i));
          s[k][1] += (unsigned long long) (x1 * __ldg (tab + k * n + i + 1));
        }
      }
      int ic[4];
      if (LIN) {
        ic[0] = ic[2] = linear_coeff_int (frac, L.out_step, 31);
        ic[1] = ic[3] = 2147483647 - ic[0];
      } else
        cubic_coeff_s32 (frac, L.out_step, ic);
      unsigned long long acc = 0;
#pragma unroll
      for (int k = 0; k < ROWS; k++)
#pragma unroll
        for (int l = 0; l < 2; l++)
          acc += (unsigned long long) ((long long) (int) (unsigned) (s[k][l] >> 31) * (long long) ic[k]);
      io.template store<int> (L, (size_t) o * L.channels + c, ars_round_s32 (acc));
    }
  } else {
    const double *tab = (const double *) L.table + row0;
    if (L.full) {                 // inner_product_gdouble_full_1_sse2
      double s0 = 0.0, s1 = 0.0;
      for (int i = 0; i < n; i += 2) {
        s0 = __dadd_rn (s0, __dmul_rn (io.template load<double> (L, idx + i, c), __ldg (tab + i)));
        s1 = __dadd_rn (s1, __dmul_rn (io.template load<double> (L, idx + i + 1, c), __ldg (tab + i + 1)));
      }
      io.template store<double> (L, (size_t) o * L.channels + c, __dadd_rn (s0, s1));
    } else if (LIN) {             // inner_product_gdouble_linear_1_sse2 (audio-resampler-x86-sse2.c:195-220)
      double s[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
      for (int i = 0; i < n; i += 2) {
        const double x0 = io.template load<double> (L, idx + i, c), x1 = io.template load<double> (L, idx + i + 1, c);
#pragma unroll
        for (int k = 0; k < 2; k++) {
          s[k][0] = __dadd_rn (s[k][0], __dmul_rn (x0, __ldg (tab + k * n + i)));
          s[k][1] = __dadd_rn (s[k][1], __dmul_rn (x1, __ldg (tab + k * n + i + 1)));
        }
      }
      const double x = __ddiv_rn ((double) frac, (double) L.out_step);      // make_coeff_gdouble_linear: ic[0]
      const double l0 = __dadd_rn (__dmul_rn (__dsub_rn (s[0][0], s[1][0]), x), s[1][0]);
      const double l1 = __dadd_rn (__dmul_rn (__dsub_rn (s[0][1], s[1][1]), x), s[1][1]);
      io.template store<double> (L, (size_t) o * L.channels + c, __dadd_rn (l0, l1));
    } else {                      // inner_product_gdouble_cubic_1_sse2
      double s[4][2];
#pragma unroll
      for (int k = 0; k < 4; k++) s[k][0] = s[k][1] = 0.0;
      for (int i = 0; i < n; i += 2) {
        const double x0 = io.template load<double> (L, idx + i, c), x1 = io.template load<double> (L, idx + i + 1, c);
#pragma unroll
        for (int k = 0; k < 4; k++) {
          s[k][0] = __dadd_rn (s[k][0], __dmul_rn (x0, __ldg (tab + k * n + i)));
          s[k][1] = __dadd_rn (s[k][1], __dmul_rn (x1, __ldg (tab + k * n + i + 1)));
        }
      }
      // make_coeff_gdouble_cubic: float literals promoted to double
      const double x = __ddiv_rn ((double) frac, (double) L.out_step), x2 = __dmul_rn (x, x), x3 = __dmul_rn (x2, x);
      const double ic0 = __dmul_rn ((double) 0.16667f, __dsub_rn (x3, x));
      const double ic1 = __dadd_rn (x, __dmul_rn ((double) 0.5f, __dsub_rn (x2, x3)));
      const double ic3 = __dsub_rn (__dadd_rn (__dmul_rn ((double) -0.33333f, x), __dmul_rn ((double) 0.5f, x2)),
          __dmul_rn ((double) 0.16667f, x3));
      const double ic2 = __dsub_rn (__dsub_rn (__dsub_rn (1.0, ic0), ic1), ic3);
      double l[2];
#pragma unroll
      for (int j = 0; j < 2; j++)
        l[j] = __dadd_rn (__dadd_rn (__dmul_rn (s[0][j], ic0), __dmul_rn (s[1][j], ic1)),
            __dadd_rn (__dmul_rn (s[2][j], ic2), __dmul_rn (s[3][j], ic3)));
      io.template store<double> (L, (size_t) o * L.channels + c, __dadd_rn (l[0], l[1]));
    }
  }
}

// The resampler in S32 / F64 (its history) over the caller's own samples (ArsLaunchX) or over packed ones (ArsLaunchP:
// unpacked on load, quantized and packed on store; the launch's descriptor is uniform across the grid)
struct ArsLaunchP {
  ArsLaunchX x;
  ArsIo io;
};

template <int FMT, bool LIN>
__global__ void __launch_bounds__ (ARS_THREADS)
ars_direct_kernel (const ArsLaunchX L)
{
  ars_direct_body<FMT, LIN> (L, ArsPlainIo ());
}

template <int FMT, bool LIN>
__global__ void __launch_bounds__ (ARS_THREADS)
ars_direct_kernel_packed (const ArsLaunchP L)
{
  ars_direct_body<FMT, LIN> (L.x, ArsPackedIo {L.io});
}

// resample-method nearest / linear / cubic: a handful of taps per output (2, 4, or those scaled by the decimation
// ratio; any count, odd ones included), FULL mode.  The reference's SIMD inner products run past n_taps into the zero
// taps every table row ends with (TAPS_OVERREAD, audio-resampler.c:34), which changes no sum, so the lanes here simply
// stop at n_taps: F32 four lanes by tap index mod 4 and (l0 + l2) + (l1 + l3) (inner_product_gfloat_full_1_sse), F64 two
// lanes by parity, the integer sums exact.  Nearest copies the first sample of the window
// (inner_product_<type>_nearest_1_c :602-612).  Warp = one output frame x 32 channels.
template <int FMT, class IO>
__device__ __forceinline__ void ars_small_body (const ArsLaunchX & L, int nearest, const IO & io)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long o = (long long) blockIdx.x * (ARS_THREADS / 32) + warp;
  if (o >= L.out_frames) return;
  const int c = blockIdx.y * 32 + lane;
  if (c >= L.channels) return;
  const long long t0 = (long long) L.samp_phase + o * L.samp_frac;
  const long long idx = (long long) L.samp_index + o * L.samp_inc + t0 / L.out_step;
  const int phase = (int) (t0 % L.out_step), n = L.n_taps;
  const size_t at = (size_t) o * L.channels + c, row0 = (size_t) phase * n;
  if (FMT == ARS_S16) {
    if (nearest) { io.template store<short> (L, at, io.template load<short> (L, idx, c)); return; }
    const short *tab = (const short *) L.table + row0;
    unsigned sum = 0;
    for (int i = 0; i < n; i++) sum += (unsigned) ((int) io.template load<short> (L, idx + i, c) * (int) __ldg (tab + i));
    io.template store<short> (L, at, (short) ars_round_s16 (sum));
  } else if (FMT == ARS_S32) {
    if (nearest) { io.template store<int> (L, at, io.template load<int> (L, idx, c)); return; }
    const int *tab = (const int *) L.table + row0;
    unsigned long long sum = 0;
    for (int i = 0; i < n; i++) sum += (unsigned long long) ((long long) io.template load<int> (L, idx + i, c) * __ldg (tab + i));
    io.template store<int> (L, at, ars_round_s32 (sum));
  } else if (FMT == ARS_F64) {
    if (nearest) { io.template store<double> (L, at, io.template load<double> (L, idx, c)); return; }
    const double *tab = (const double *) L.table + row0;
    double s0 = 0.0, s1 = 0.0;
    for (int i = 0; i < n; i += 2) {
      s0 = __dadd_rn (s0, __dmul_rn (io.template load<double> (L, idx + i, c), __ldg (tab + i)));
      if (i + 1 < n) s1 = __dadd_rn (s1, __dmul_rn (io.template load<double> (L, idx + i + 1, c), __ldg (tab + i + 1)));
    }
    io.template store<double> (L, at, __dadd_rn (s0, s1));
  } else {
    if (nearest) { io.template store<float> (L, at, io.template load<float> (L, idx, c)); return; }
    const float *tab = (const float *) L.table + row0;
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i = 0; i < n; i += 4)
#pragma unroll
      for (int l = 0; l < 4; l++)
        if (i + l < n) s[l] = __fadd_rn (s[l], __fmul_rn (io.template load<float> (L, idx + i + l, c), __ldg (tab + i + l)));
    io.template store<float> (L, at, ars_lane_sum (s));
  }
}

template <int FMT>
__global__ void __launch_bounds__ (ARS_THREADS)
ars_small_kernel (const ArsLaunchX L, int nearest)
{
  ars_small_body<FMT> (L, nearest, ArsPlainIo ());
}

template <int FMT>
__global__ void __launch_bounds__ (ARS_THREADS)
ars_small_kernel_packed (const ArsLaunchP L, int nearest)
{
  ars_small_body<FMT> (L.x, nearest, ArsPackedIo {L.io});
}

// new history = frames [first, first+keep) of the (old history ++ input) stream, any sample width
template <typename T>
__device__ __forceinline__ void ars_history_copy (T *dst, const T *hist, const T *in, long long hist_frames,
    long long first, long long keep, int channels)
{
  const long long n = keep * channels;
  for (long long i = blockIdx.x * (long long) blockDim.x + threadIdx.x; i < n; i += (long long) gridDim.x * blockDim.x) {
    const long long f = first + i / channels;
    const int c = (int) (i % channels);
    T v = 0;
    if (f < hist_frames) v = hist[f * channels + c];
    else if (in) v = in[(f - hist_frames) * channels + c];
    dst[i] = v;
  }
}

// the kernels keep their names (F32 and S32 samples: ars_history_kernel), which the launch records pin
template <typename T>
__global__ void ars_history_kernel_x (T *dst, const T *hist, const T *in, long long hist_frames, long long first, long long keep, int channels)
{
  ars_history_copy (dst, hist, in, hist_frames, first, keep, channels);
}
__global__ void ars_history_kernel (float *dst, const float *hist, const float *in, long long hist_frames, long long first, long long keep,
    int channels)
{
  ars_history_copy (dst, hist, in, hist_frames, first, keep, channels);
}
// the same for packed input: the kept input samples are unpacked into the history, which holds T (int: S32, double: F64)
template <typename T>
__global__ void ars_history_kernel_packed (T *dst, const T *hist, const unsigned char *in, ArsIo io, long long hist_frames,
    long long first, long long keep, int channels)
{
  const long long n = keep * channels;
  for (long long i = blockIdx.x * (long long) blockDim.x + threadIdx.x; i < n; i += (long long) gridDim.x * blockDim.x) {
    const long long f = first + i / channels;
    const int c = (int) (i % channels);
    T v = 0;
    if (f < hist_frames) v = hist[f * channels + c];
    else if (in) {
      const unsigned char *p = in + (size_t) ((f - hist_frames) * channels + c) * io.step;
      v = sizeof (T) == 8 ? (T) ars_unpack_f64 (io, p) : (T) ars_unpack_int (io, p);
    }
    dst[i] = v;
  }
}

}  // namespace b200

using namespace b200;

// Tensor map of the caller's input for the pipelined kernel's window copies: 2-D [frames][channels] F32, box = cb channels x
// win frames, out-of-bounds rows read as zeros.  Encoded on the host per call (the input pointer changes with every buffer;
// cuTensorMapEncodeTiled is pure CPU work) through the driver entry point - the library does not link libcuda.
// Returns 1 when the map is usable.
#ifndef B200_CUDA_EMU
static_assert (sizeof (ArsTensorMap) == sizeof (CUtensorMap), "CUtensorMap is 128 bytes");
typedef CUresult (*ars_encode_fn) (CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static int ars_encode_window_map (ArsTensorMap *tm, const void *in, unsigned long long in_frames, int channels, int cb, int win, int elem_bytes = 4)
{
  static ars_encode_fn fn = [] () -> ars_encode_fn {
    void *f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint ("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
    return (ars_encode_fn) f;
  } ();
  if (!fn || !in || in_frames == 0 || win > 256 || cb > 256 || (((uintptr_t) in) & 15) || (channels & 3)) return 0;
  const cuuint64_t gdim[2] = {(cuuint64_t) channels, (cuuint64_t) in_frames};
  const cuuint64_t gstride[1] = {(cuuint64_t) channels * (cuuint64_t) elem_bytes};
  const cuuint32_t box[2] = {(cuuint32_t) cb, (cuuint32_t) win}, estr[2] = {1, 1};
  if (((cuuint64_t) channels * (cuuint64_t) elem_bytes) & 15) return 0;
  const CUresult r = fn ((CUtensorMap *) tm, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *) in, gdim, gstride, box, estr,
      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}
#else
static int ars_encode_window_map (ArsTensorMap *, const void *, unsigned long long, int, int, int, int = 4) { return 0; }
#endif

// A/B and tuning switches of the resampler (README, environment knobs), read once when a handle is created
struct ArsKnobs {
  bool generic = false;          // B200_ARS_GENERIC: S16 runs ars_direct_kernel, F32 FULL ars_full_kernel
  bool nopipe = false;           // B200_ARS_NOPIPE: no persistent pipeline
  bool pipe_v1 = false;          // B200_ARS_PIPE_V1: the cp.async form of the F32 pipeline
  bool no_tensormap = false;     // B200_ARS_NO_TENSORMAP: the pipelines' window copies row by row
  int no = 32;                   // B200_ARS_NO: outputs per CTA of the F32 tile / generic kernel (4 .. 64, a power of two)
  int cb = 0, cpt = 0;           // B200_ARS_CB (32, 64: at most this many channels per F32 tile CTA), B200_ARS_CPT (1, 4)
  int grid = 0;                  // B200_ARS_GRID: at most this many persistent CTAs
};

static ArsKnobs ars_read_knobs ()
{
  ArsKnobs k;
  k.generic = getenv ("B200_ARS_GENERIC") != nullptr;
  k.nopipe = getenv ("B200_ARS_NOPIPE") != nullptr;
  k.pipe_v1 = getenv ("B200_ARS_PIPE_V1") != nullptr;
  k.no_tensormap = getenv ("B200_ARS_NO_TENSORMAP") != nullptr;
  const char *no = getenv ("B200_ARS_NO"), *cb = getenv ("B200_ARS_CB"), *cpt = getenv ("B200_ARS_CPT"), *grid = getenv ("B200_ARS_GRID");
  if (no && atoi (no) >= ARS_RQ && atoi (no) <= 64 && !(atoi (no) & (atoi (no) - 1))) k.no = atoi (no);   // s_rel/s_phase hold 64
  if (cb && (atoi (cb) == 32 || atoi (cb) == 64)) k.cb = atoi (cb);
  if (cpt && (atoi (cpt) == 1 || atoi (cpt) == 4)) k.cpt = atoi (cpt);
  if (grid && atoi (grid) > 0) k.grid = atoi (grid);
  return k;
}

// the kernel one b200_ars_process call runs (DESIGN.md §4.5)
enum ArsKern { ARS_K_SMALL, ARS_K_DIRECT, ARS_K_INTERP, ARS_K_FULL, ARS_K_TILE, ARS_K_TILE_S16, ARS_K_PIPE, ARS_K_PIPE_V1, ARS_K_PIPE_S16 };

struct ArsRoute {
  int status = B200_OK;          // B200_ERR_UNSUPPORTED: ars_full_kernel's tap rows do not fit in shared memory
  ArsKern kern = ARS_K_SMALL;
  int no = 0;                    // outputs per CTA (tile, pipeline and generic kernels)
  int cb = 0, cpt = 0;           // channels per CTA (ars_full_kernel: 32 x warps across channels), per thread (F32 tile)
  ArsTile tile = ArsTile ();     // win and nch (tile and pipeline kernels)
  size_t smem = 0;               // dynamic shared memory
};

// floats per staged tap row of ars_full_kernel: the taps shifted by up to 3, padded to a multiple of 4
static int ars_row_pitch (const ArsPlan & p) { return (p.n_taps + 4 + 3) & ~3; }

// smem_optin: the device's opt-in shared memory per block; aligned16: history, input and output are 16-byte aligned
static ArsRoute ars_select_route (const ArsPlan & p, const ArsKnobs & k, int smem_optin, bool aligned16)
{
  if (p.small || p.copy) return {B200_OK, ARS_K_SMALL};
  // the persistent pipelines: whole 128-channel blocks, 16-byte aligned streams, both stages in shared memory
  const ArsTile pt = ars_tile_geometry (p, ARS_PIPE_NO);
  const size_t pipe_smem = 2 * ars_tile_smem (pt, ARS_PIPE_NO, ARS_PIPE_CB, p.bps);
  const bool pipe = (p.channels % ARS_PIPE_CB) == 0 && !k.generic && !k.nopipe && aligned16 && pipe_smem + 2048 <= (size_t) smem_optin;
  if (p.fmt == ARS_S16 && p.full && !k.generic) {
    if (pipe) return {B200_OK, ARS_K_PIPE_S16, ARS_PIPE_NO, ARS_PIPE_CB, 0, pt, pipe_smem};
    // the tile kernel: the F32 tile geometry with 4-byte staged samples and taps
    const int no = 32, cb = p.channels >= 128 ? 128 : 64;
    const ArsTile t = ars_tile_geometry (p, no);
    const size_t smem = ars_tile_smem (t, no, cb, 4);
    if (p.channels >= 64 && smem <= (size_t) ARS_TILE_SMEM) return {B200_OK, ARS_K_TILE_S16, no, cb, 0, t, smem};
  }
  if (p.fmt != ARS_F32) return {B200_OK, ARS_K_DIRECT};
  if (!p.full) return {B200_OK, ARS_K_INTERP};
  const size_t row_bytes = (size_t) ars_row_pitch (p) * sizeof (float);
  int no = k.no;                                                 // 32 by default: measured best for the tile kernel (3 CTAs / SM)
  while (no > ARS_RQ && no * row_bytes > 96 * 1024) no >>= 1;
  if (no * row_bytes > 160 * 1024) return {B200_ERR_UNSUPPORTED};
  if (pipe) return {B200_OK, k.pipe_v1 ? ARS_K_PIPE_V1 : ARS_K_PIPE, ARS_PIPE_NO, ARS_PIPE_CB, 0, pt, pipe_smem};
  int wcn = std::min ((p.channels + 31) / 32, 8);
  while (8 % wcn) wcn++;                                         // 1, 2, 4 or 8 warps across channels
  // the tile kernel when the CTA's input window fits in shared memory next to the chunk-major taps: 2 channels per thread
  int cb = 32 * std::min (wcn, 4);
  if (k.cb && k.cb < cb) cb = k.cb;
  int cpt = cb >= 64 ? 2 : 1;
  if (k.cpt == 1 || (k.cpt == 4 && cb >= 128)) cpt = k.cpt;
  const ArsTile t = ars_tile_geometry (p, no);
  const size_t smem = ars_tile_smem (t, no, cb, 4);
  if (smem <= (size_t) ARS_TILE_SMEM && !k.generic) return {B200_OK, ARS_K_TILE, no, cb, cpt, t, smem};
  return {B200_OK, ARS_K_FULL, no, 32 * wcn, 0, ArsTile (), no * row_bytes};
}

struct b200_ars {
  ArsPlan plan;
  int device = -1;
  b200_ars_config cfg;           // as created / last updated (b200_ars_update re-designs the filter from it)
  ArsKnobs knobs;
  int smem_optin = 0, sms = 0;   // the device's opt-in shared memory per block and its SM count
  float *d_phases = nullptr;
  float *d_qtab = nullptr;       // chunk-major taps of every 4-output group (F32 FULL; S16 FULL in whole 128-channel blocks)
  float *d_proto = nullptr;      // interpolated mode: the oversampled prototype rows
  void *d_table_x = nullptr;     // other sample formats: phase taps (FULL) or prototype rows, in the samples' type
  float *d_hist[2] = {nullptr, nullptr};
  size_t hist_cap[2] = {0, 0};   // frames
  int cur = 0;
  // reference state (audio-resampler-private.h:103-112)
  int samp_index = 0, samp_phase = 0, skip = 0;
  size_t samples_avail = 0;
  // system-memory peers (b200_ars_process_host*)
  static const int kSlots = 3;
  HostRing<kSlots> ring;
};

static int ars_reset_state (b200_ars * h, cudaStream_t stream)
{
  h->samp_index = 0;
  h->samples_avail = h->plan.n_taps / 2 - 1;                    // gst_audio_resampler_reset, :1465-1484
  if (h->device >= 0 && h->d_hist[h->cur])
    B200_CUDA_TRY (cudaMemsetAsync (h->d_hist[h->cur], 0, (size_t) (h->plan.n_taps / 2) * h->plan.channels * h->plan.bps, stream));
  return B200_OK;
}

// `stream` is the stream the next writers / readers of the buffer run on: the clear is ordered there, not on the legacy
// default stream (a cudaStreamNonBlocking user stream is not ordered against that one)
static int ars_ensure_hist (b200_ars * h, int which, size_t frames, cudaStream_t stream)
{
  if (h->hist_cap[which] >= frames) return B200_OK;
  size_t cap = frames + (size_t) h->plan.n_taps;
  float *n = nullptr;
  const size_t bps = (size_t) h->plan.bps;                        // the buffers hold samples of the plan's format
  B200_CUDA_TRY (cudaMalloc ((void **) &n, cap * h->plan.channels * bps));
  B200_CUDA_TRY (cudaMemsetAsync (n, 0, cap * h->plan.channels * bps, stream));
  if (h->d_hist[which]) {
    if (which == h->cur && h->samples_avail)
      B200_CUDA_TRY (cudaMemcpyAsync (n, h->d_hist[which], h->samples_avail * h->plan.channels * bps, cudaMemcpyDeviceToDevice, stream));
    B200_CUDA_TRY (cudaStreamSynchronize (stream));                 // the old buffer is released below
    cudaFree (h->d_hist[which]);
  }
  h->d_hist[which] = n;
  h->hist_cap[which] = cap;
  return B200_OK;
}

// the plan's tables on the device (the current device is the handle's): phase taps or prototype rows, and for the tile and
// pipeline kernels the pre-laid chunk-major rows
static int ars_upload_tables (b200_ars * h)
{
  int st;
  const ArsPlan & q = h->plan;
  cudaFree (h->d_phases); cudaFree (h->d_qtab); cudaFree (h->d_proto); cudaFree (h->d_table_x);
  h->d_phases = h->d_qtab = h->d_proto = nullptr; h->d_table_x = nullptr;
  if (q.fmt != ARS_F32) {
    const std::vector<uint8_t> & t = q.full ? q.phases_x : q.proto_x;
    uint8_t *d = nullptr;
    st = upload (&d, t.data (), t.size ());
    h->d_table_x = d;
  } else
    st = q.full ? upload (&h->d_phases, q.phases.data (), q.phases.size ()) : upload (&h->d_proto, q.proto.data (), q.proto.size ());
  // tap rows of every (alignment, phase) group: F32 for the tile kernels and the pipeline, S16 (32-bit ints in the F32
  // layout) for its pipeline; bounded by the FULL-mode threshold (bps * n_taps * out_rate < 1 MiB  =>  at most 16 x that)
  if (st == B200_OK && q.full && !q.small && !q.copy && (q.fmt == ARS_F32 || (q.fmt == ARS_S16 && (q.channels % ARS_PIPE_CB) == 0))) {
    std::vector<float> tab;
    const int nch = ars_tile_geometry (q, 0).nch;
    if (q.fmt == ARS_F32) ars_build_qtab<float, float> (q, q.phases.data (), nch, &tab);
    else ars_build_qtab<int16_t, int32_t> (q, (const int16_t *) q.phases_x.data (), nch, &tab);
    st = upload (&h->d_qtab, tab.data (), tab.size ());
  }
  return st;
}

extern "C" {

int b200_ars_create (const b200_ars_config * cfg, int device, b200_ars ** handle)
{
  if (!cfg || !handle) return B200_ERR_INVALID_ARG;
  *handle = nullptr;
  b200_ars *h = new (std::nothrow) b200_ars ();
  if (!h) return B200_ERR_NOMEM;
  h->cfg = *cfg;
  int st = build_ars_plan (*cfg, &h->plan);
  if (st != B200_OK) { delete h; return st; }
  h->device = device;
  h->knobs = ars_read_knobs ();
  h->samples_avail = h->plan.n_taps / 2 - 1;
  if (device >= 0) {
    int n = b200_device_count ();
    if (n <= 0) { delete h; return n < 0 ? n : B200_ERR_NO_DEVICE; }
    if (device >= n) { delete h; return B200_ERR_INVALID_ARG; }
    DeviceGuard g (device);
    h->sms = sm_count (device);
    st = ars_upload_tables (h);
    if (st == B200_OK) st = ars_ensure_hist (h, 0, (size_t) h->plan.n_taps, nullptr);
    if (st == B200_OK) st = ars_ensure_hist (h, 1, (size_t) h->plan.n_taps, nullptr);
    if (st == B200_OK && cudaDeviceSynchronize () != cudaSuccess) st = B200_ERR_CUDA;   // clears done before any user stream
    if (st == B200_OK && cudaDeviceGetAttribute (&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess)
      st = B200_ERR_CUDA;
    // the dynamic shared memory each kernel the route can pick may ask for; 0: the device's opt-in maximum
    const struct { const void *fn; int bytes; } smem[] = {
      {(const void *) ars_full_kernel, 160 * 1024}, {(const void *) ars_pipe_kernel, 0}, {(const void *) ars_pipe_kernel_v1, 0},
      {(const void *) ars_pipe_kernel_s16, 0}, {(const void *) ars_tile_kernel<128, 4>, ARS_TILE_SMEM},
      {(const void *) ars_tile_kernel<128, 2>, ARS_TILE_SMEM}, {(const void *) ars_tile_kernel<128, 1>, ARS_TILE_SMEM},
      {(const void *) ars_tile_kernel<64, 2>, ARS_TILE_SMEM}, {(const void *) ars_tile_kernel<64, 1>, ARS_TILE_SMEM},
      {(const void *) ars_tile_kernel<32, 1>, ARS_TILE_SMEM}, {(const void *) ars_tile_kernel_s16<128>, ARS_TILE_SMEM},
      {(const void *) ars_tile_kernel_s16<64>, ARS_TILE_SMEM}};
    for (size_t i = 0; st == B200_OK && i < sizeof (smem) / sizeof (smem[0]); i++) {
      if (smem[i].bytes) cudaFuncSetAttribute (smem[i].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem[i].bytes);
      else st = allow_max_dyn_smem (smem[i].fn);
    }
    if (st != B200_OK) {
      b200_ars_destroy (h);
      return st;
    }
  }
  *handle = h;
  return B200_OK;
}

void b200_ars_destroy (b200_ars * h)
{
  if (!h) return;
  if (h->device >= 0) {
    DeviceGuard g (h->device);
    cudaFree (h->d_phases); cudaFree (h->d_qtab); cudaFree (h->d_proto); cudaFree (h->d_table_x); cudaFree (h->d_hist[0]); cudaFree (h->d_hist[1]);
    h->ring.drain ();
    h->ring.release ();
  }
  delete h;
}

int b200_ars_reset (b200_ars * h)
{
  if (!h) return B200_ERR_INVALID_ARG;
  if (h->device >= 0) {
    DeviceGuard g (h->device);
    // flush / discont: wait for whatever stream the caller last processed on, clear, and wait for the clear - the next
    // process() may come on a non-blocking stream that the legacy stream does not order
    B200_CUDA_TRY (cudaDeviceSynchronize ());
    int st = ars_reset_state (h, nullptr);
    if (st != B200_OK) return st;
    B200_CUDA_TRY (cudaStreamSynchronize (nullptr));
    return B200_OK;
  }
  return ars_reset_state (h, nullptr);
}

// gst_audio_resampler_update () as the element drives it (gst_audio_resample_update_state, gstaudioresample.c:398-437:
// new rates AND a fresh option bag -> the filter is re-designed): the phase is rescaled to the new output rate, the rates'
// common divisor is reduced only while the phase error stays below DEFAULT_OPT_MAX_PHASE_ERROR 0.1
// (audio-resampler.c:1517-1551), and when the tap count changes the history moves by half the difference (:1572-1603) -
// shrinking drops the oldest samples, growing leaves the oldest ones in place twice.  The stream position survives.
// One corner is NOT the reference's: when the tap count grows by more than twice the kept history, the reference's
// "old samples left in place" (its FIXME, :1597-1599) are leftover bytes of earlier calls in its sample buffer; the
// product has zeros there.
int b200_ars_update (b200_ars * h, int in_rate, int out_rate)
{
  if (!h) return B200_ERR_INVALID_ARG;
  if (in_rate <= 0) in_rate = h->plan.in_step;                     // "0 = unchanged" means the REDUCED rate, like the reference
  if (out_rate <= 0) out_rate = h->plan.out_step;
  long long sp = (long long) ((unsigned long long) h->samp_phase * (unsigned long long) out_rate / (unsigned long long) h->plan.out_step);
  int a = in_rate, b = out_rate;
  while (b) { int t = a; a = b; b = t % b; }
  int g = a;
  while (g > 1) {
    const double ph1 = (double) sp / out_rate, ph2 = (double) (sp / g) / (out_rate / g);
    if (fabs (ph1 - ph2) < 0.1) break;
    int factor = 2;
    while (g % factor != 0) factor++;
    g /= factor;
  }
  b200_ars_config cfg = h->cfg;
  cfg.in_rate = in_rate; cfg.out_rate = out_rate;
  ArsPlan np;
  int st = build_ars_plan (cfg, &np, g);
  if (st != B200_OK) return st;
  const int old_taps = h->plan.n_taps;
  const int diff = (np.n_taps - old_taps) / 2;
  if (h->device >= 0) {
    DeviceGuard dg (h->device);
    if (!dg.ok) return B200_ERR_CUDA;
    B200_CUDA_TRY (cudaDeviceSynchronize ());                      // kernels of the old filter still read its tables
    if (diff != 0) {
      // history into the other buffer, shifted (samp_index is 0 between calls: process () compacts)
      const size_t bpf = (size_t) np.channels * np.bps;
      const size_t avail = h->samples_avail;
      const long long new_avail = (long long) avail + diff;
      const int nxt = h->cur ^ 1;
      ArsPlan keep = h->plan;
      h->plan = np;                                                // ars_ensure_hist sizes with the new tap count
      st = ars_ensure_hist (h, nxt, (size_t) std::max (new_avail, (long long) avail) + 1, nullptr);
      if (st != B200_OK) { h->plan = keep; return st; }
      const uint8_t *src = (const uint8_t *) h->d_hist[h->cur];
      uint8_t *dst = (uint8_t *) h->d_hist[nxt];
      if (diff < 0) {
        if (new_avail > 0)
          B200_CUDA_TRY (cudaMemcpy (dst, src + (size_t) (-diff) * bpf, (size_t) new_avail * bpf, cudaMemcpyDeviceToDevice));
      } else {
        const size_t lead = std::min ((size_t) diff, avail);      // "just leave the old samples in there"
        if (lead) B200_CUDA_TRY (cudaMemcpy (dst, src, lead * bpf, cudaMemcpyDeviceToDevice));
        if (avail) B200_CUDA_TRY (cudaMemcpy (dst + (size_t) diff * bpf, src, avail * bpf, cudaMemcpyDeviceToDevice));
      }
      h->cur = nxt;
      h->samples_avail = (size_t) std::max (new_avail, 0LL);
    } else
      h->plan = np;
    if ((st = ars_upload_tables (h)) != B200_OK) return st;
    B200_CUDA_TRY (cudaDeviceSynchronize ());
  } else {
    h->plan = np;
    h->samples_avail = (size_t) std::max ((long long) h->samples_avail + diff, 0LL);
  }
  h->cfg = cfg;
  h->samp_phase = (int) (sp / g);
  return B200_OK;
}

size_t b200_ars_get_out_frames (b200_ars * h, size_t in_frames)
{
  if (!h) return 0;
  const ArsPlan & p = h->plan;
  const size_t need = (size_t) p.n_taps + h->samp_index + h->skip, avail = h->samples_avail + in_frames;
  if (avail < need) return 0;
  size_t out = (avail - need) * p.out_step;
  if (out < (size_t) h->samp_phase) return 0;
  return (out - h->samp_phase) / p.in_step + 1;
}

size_t b200_ars_get_in_frames (b200_ars * h, size_t out_frames)
{
  if (!h) return 0;
  const ArsPlan & p = h->plan;
  return (h->samp_phase + out_frames * p.samp_frac) / p.out_step + out_frames * p.samp_inc;
}

size_t b200_ars_get_max_latency (b200_ars * h) { return h ? h->plan.n_taps / 2 : 0; }

int b200_ars_process (b200_ars * h, const void *in_v, size_t in_frames, void *out_v,
    size_t out_capacity_frames, size_t * out_frames_ret, void *cuda_stream)
{
  const float *in = (const float *) in_v;
  float *out = (float *) out_v;
  if (!h || (!out && out_capacity_frames)) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  cudaStream_t stream = (cudaStream_t) cuda_stream;
  const ArsPlan & p = h->plan;
  size_t out_frames = b200_ars_get_out_frames (h, in_frames);
  if (out_frames > out_capacity_frames) out_frames = out_capacity_frames;
  if (out_frames_ret) *out_frames_ret = out_frames;
  // gst_audio_resampler_resample (audio-resampler.c:1750-1805)
  if ((size_t) h->skip >= in_frames) { h->skip -= (int) in_frames; return B200_OK; }
  h->samp_index += h->skip;
  const size_t hist = h->samples_avail, avail = hist + in_frames;
  const size_t need = (size_t) p.n_taps + h->samp_index;
  size_t consumed = 0;
  long long moved_from = 0;       // the absolute sample index the reference's buffers are shifted down by (macros.h:91-93)
  int new_phase = h->samp_phase;
  if (avail >= need && out_frames > 0) {
    const bool aligned16 = ((((uintptr_t) h->d_hist[h->cur]) | ((uintptr_t) in_v) | ((uintptr_t) out_v)) & 15) == 0;
    const ArsRoute r = ars_select_route (p, h->knobs, h->smem_optin, aligned16);
    if (r.status != B200_OK) return r.status;
    ArsLaunch L;
    L.hist = h->d_hist[h->cur]; L.in = in; L.out = out;
    L.phases = r.kern == ARS_K_TILE_S16 ? (const float *) h->d_table_x : h->d_phases;
    L.hist_frames = (long long) hist; L.avail = (long long) avail; L.out_frames = (long long) out_frames;
    L.channels = p.channels; L.n_taps = p.n_taps; L.out_step = p.out_step;
    L.samp_inc = p.samp_inc; L.samp_frac = p.samp_frac;
    L.samp_index = h->samp_index; L.samp_phase = h->samp_phase;
    L.no = r.no; L.wcn = r.cb / 32; L.row_pitch = ars_row_pitch (p);
    ArsLaunchX X;
    X.hist = L.hist; X.in = in_v; X.out = out_v;
    X.table = p.fmt == ARS_F32 ? (const void *) h->d_phases : (const void *) h->d_table_x;
    X.hist_frames = L.hist_frames; X.avail = L.avail; X.out_frames = L.out_frames;
    X.channels = p.channels; X.n_taps = p.n_taps; X.out_step = p.out_step;
    X.samp_inc = p.samp_inc; X.samp_frac = p.samp_frac; X.samp_index = h->samp_index; X.samp_phase = h->samp_phase;
    X.full = p.full ? 1 : 0; X.oversample = p.oversample;
    ArsTile T = r.tile;
    T.qtab = (const float4 *) h->d_qtab;
    // one warp per output frame x 32 channels; the tile and generic kernels: no outputs x cb channels per CTA
    const dim3 warps ((unsigned) ((out_frames + ARS_THREADS / 32 - 1) / (ARS_THREADS / 32)), (unsigned) ((p.channels + 31) / 32));
    auto tiles = [&] { return dim3 ((unsigned) ((out_frames + r.no - 1) / r.no), (unsigned) ((p.channels + r.cb - 1) / r.cb)); };
    const int nearest = p.small == B200_ARS_METHOD_NEAREST || p.copy;
    const bool lin = p.linear && !p.full;
    // packed samples reach only the S32 / F64 routes: the small and direct kernels
    const ArsLaunchP P = {X, p.io};
    if (p.io.kind != ARS_IO_NONE && r.kern == ARS_K_SMALL) {
      if (p.fmt == ARS_S32) ars_small_kernel_packed<ARS_S32> <<<warps, ARS_THREADS, 0, stream>>> (P, nearest);
      else ars_small_kernel_packed<ARS_F64> <<<warps, ARS_THREADS, 0, stream>>> (P, nearest);
    } else if (p.io.kind != ARS_IO_NONE) {
      if (p.fmt == ARS_S32 && lin) ars_direct_kernel_packed<ARS_S32, true> <<<warps, ARS_THREADS, 0, stream>>> (P);
      else if (p.fmt == ARS_S32) ars_direct_kernel_packed<ARS_S32, false> <<<warps, ARS_THREADS, 0, stream>>> (P);
      else if (lin) ars_direct_kernel_packed<ARS_F64, true> <<<warps, ARS_THREADS, 0, stream>>> (P);
      else ars_direct_kernel_packed<ARS_F64, false> <<<warps, ARS_THREADS, 0, stream>>> (P);
    } else
    switch (r.kern) {
      case ARS_K_SMALL:
        if (p.fmt == ARS_S16) ars_small_kernel<ARS_S16> <<<warps, ARS_THREADS, 0, stream>>> (X, nearest);
        else if (p.fmt == ARS_S32) ars_small_kernel<ARS_S32> <<<warps, ARS_THREADS, 0, stream>>> (X, nearest);
        else if (p.fmt == ARS_F64) ars_small_kernel<ARS_F64> <<<warps, ARS_THREADS, 0, stream>>> (X, nearest);
        else ars_small_kernel<ARS_F32> <<<warps, ARS_THREADS, 0, stream>>> (X, nearest);
        break;
      case ARS_K_DIRECT:
        if (p.fmt == ARS_S16 && lin) ars_direct_kernel<ARS_S16, true> <<<warps, ARS_THREADS, 0, stream>>> (X);
        else if (p.fmt == ARS_S16) ars_direct_kernel<ARS_S16, false> <<<warps, ARS_THREADS, 0, stream>>> (X);
        else if (p.fmt == ARS_S32 && lin) ars_direct_kernel<ARS_S32, true> <<<warps, ARS_THREADS, 0, stream>>> (X);
        else if (p.fmt == ARS_S32) ars_direct_kernel<ARS_S32, false> <<<warps, ARS_THREADS, 0, stream>>> (X);
        else if (lin) ars_direct_kernel<ARS_F64, true> <<<warps, ARS_THREADS, 0, stream>>> (X);
        else ars_direct_kernel<ARS_F64, false> <<<warps, ARS_THREADS, 0, stream>>> (X);
        break;
      case ARS_K_INTERP:
        if (p.linear) ars_interp_kernel<true> <<<warps, ARS_THREADS, 0, stream>>> (L, h->d_proto, p.oversample);
        else ars_interp_kernel<false> <<<warps, ARS_THREADS, 0, stream>>> (L, h->d_proto, p.oversample);
        break;
      case ARS_K_FULL:
        ars_full_kernel <<<tiles (), ARS_THREADS, r.smem, stream>>> (L);
        break;
      case ARS_K_TILE:
        if (r.cb == 128 && r.cpt == 4) ars_tile_kernel<128, 4> <<<tiles (), ARS_THREADS, r.smem, stream>>> (L, T);
        else if (r.cb == 128 && r.cpt == 2) ars_tile_kernel<128, 2> <<<tiles (), ARS_THREADS, r.smem, stream>>> (L, T);
        else if (r.cb == 128) ars_tile_kernel<128, 1> <<<tiles (), ARS_THREADS, r.smem, stream>>> (L, T);
        else if (r.cb == 64 && r.cpt == 2) ars_tile_kernel<64, 2> <<<tiles (), ARS_THREADS, r.smem, stream>>> (L, T);
        else if (r.cb == 64) ars_tile_kernel<64, 1> <<<tiles (), ARS_THREADS, r.smem, stream>>> (L, T);
        else ars_tile_kernel<32, 1> <<<tiles (), ARS_THREADS, r.smem, stream>>> (L, T);
        break;
      case ARS_K_TILE_S16:
        if (r.cb == 128) ars_tile_kernel_s16<128> <<<tiles (), ARS_THREADS, r.smem, stream>>> (L, T);
        else ars_tile_kernel_s16<64> <<<tiles (), ARS_THREADS, r.smem, stream>>> (L, T);
        break;
      case ARS_K_PIPE: case ARS_K_PIPE_V1: case ARS_K_PIPE_S16: {
        // persistent CTAs walk the (64-output, 128-channel) tiles; the input's tensor map changes with every buffer
        const int n_fb = (int) ((out_frames + ARS_PIPE_NO - 1) / ARS_PIPE_NO), n_cb = p.channels / ARS_PIPE_CB;
        int grid = (int) std::min ((long long) n_fb * n_cb, (long long) h->sms);
        if (h->knobs.grid) grid = std::min (grid, h->knobs.grid);
        ArsTensorMap tm = ArsTensorMap ();
        const int use_tm = r.kern != ARS_K_PIPE_V1 && !h->knobs.no_tensormap &&
            ars_encode_window_map (&tm, in_v, (unsigned long long) in_frames, p.channels, ARS_PIPE_CB, T.win, p.width);
        if (r.kern == ARS_K_PIPE) ars_pipe_kernel <<<grid, ARS_PIPE_THREADS, r.smem, stream>>> (L, T, n_fb, n_cb, tm, use_tm);
        else if (r.kern == ARS_K_PIPE_S16) ars_pipe_kernel_s16 <<<grid, ARS_PIPE_THREADS, r.smem, stream>>> (L, T, n_fb, n_cb, tm, use_tm);
        else ars_pipe_kernel_v1 <<<grid, ARS_PIPE_THREADS, r.smem, stream>>> (L, T, n_fb, n_cb);
        break;
      }
    }
    B200_CUDA_TRY (cudaGetLastError ());
    // state after out_frames outputs (closed form of the stepping loop)
    const long long t = (long long) h->samp_phase + (long long) out_frames * p.samp_frac;
    const long long end_index = (long long) h->samp_index + (long long) out_frames * p.samp_inc + t / p.out_step;
    new_phase = (int) (t % p.out_step);
    consumed = (size_t) (end_index - h->samp_index);
    moved_from = end_index;
    h->samp_index = 0;
    h->samp_phase = new_phase;
  }
  // history: what the reference keeps in its per-channel buffers (macros.h:91-93, :1790-1804)
  size_t keep = avail;
  if (consumed > 0) {
    if (avail > consumed) keep = avail - consumed;
    else { keep = 0; h->skip = (int) (consumed - avail); }
  }
  const int nxt = h->cur ^ 1;
  int st = ars_ensure_hist (h, nxt, keep, stream);
  if (st != B200_OK) return st;
  // The reference shifts its buffers down by the ABSOLUTE final sample index but counts what is left from the index it
  // started at (consumed = final - initial, :1790-1804).  The two differ only after a skip (nearest method while
  // decimating: the next window starts beyond the data), and then the last `initial` of the kept samples are not the
  // stream's tail but whatever the shift left in place: the frames at those same buffer positions.  Part 1 = frames
  // [moved_from, ...) -> position 0, part 2 = frames [n1, keep) staying where they were (empty without a skip).
  const size_t n1 = (long long) avail > moved_from ? std::min (keep, (size_t) ((long long) avail - moved_from)) : 0;
  auto copy_hist = [&] (size_t dst_frame, long long from, size_t count) {
    if (!count) return;
    const long long n = (long long) count * p.channels;
    const int blocks = (int) ((n + 255) / 256 > 1184 ? 1184 : (n + 255) / 256);
    const size_t off = dst_frame * p.channels;
    if (p.io.kind != ARS_IO_NONE && p.bps == 8)
      ars_history_kernel_packed<double> <<<blocks, 256, 0, stream>>> ((double *) h->d_hist[nxt] + off,
          (const double *) h->d_hist[h->cur], (const unsigned char *) in_v, p.io, (long long) hist, from, (long long) count,
          p.channels);
    else if (p.io.kind != ARS_IO_NONE)
      ars_history_kernel_packed<int> <<<blocks, 256, 0, stream>>> ((int *) h->d_hist[nxt] + off,
          (const int *) h->d_hist[h->cur], (const unsigned char *) in_v, p.io, (long long) hist, from, (long long) count,
          p.channels);
    else if (p.bps == 2)
      ars_history_kernel_x<unsigned short> <<<blocks, 256, 0, stream>>> ((unsigned short *) h->d_hist[nxt] + off,
          (const unsigned short *) h->d_hist[h->cur], (const unsigned short *) in_v, (long long) hist, from,
          (long long) count, p.channels);
    else if (p.bps == 8)
      ars_history_kernel_x<unsigned long long> <<<blocks, 256, 0, stream>>> ((unsigned long long *) h->d_hist[nxt] + off,
          (const unsigned long long *) h->d_hist[h->cur], (const unsigned long long *) in_v, (long long) hist,
          from, (long long) count, p.channels);
    else
      ars_history_kernel <<<blocks, 256, 0, stream>>> (h->d_hist[nxt] + off, h->d_hist[h->cur], in, (long long) hist,
          from, (long long) count, p.channels);
  };
  copy_hist (0, moved_from, n1);
  copy_hist (n1, (long long) n1, keep - n1);
  if (keep) B200_CUDA_TRY (cudaGetLastError ());
  h->cur = nxt;
  h->samples_avail = keep;
  return B200_OK;
}

int b200_ars_get_plan_info (const b200_ars * h, b200_ars_plan_info * info)
{
  if (!h || !info) return B200_ERR_INVALID_ARG;
  info->n_taps = h->plan.n_taps; info->n_phases = h->plan.n_phases; info->in_step = h->plan.in_step;
  info->out_step = h->plan.out_step; info->filter_mode = h->plan.full ? 1 : 0; info->oversample = h->plan.oversample;
  return B200_OK;
}

int b200_ars_get_phase_taps (const b200_ars * h, int phase, float *taps, size_t len)
{
  if (!h || !taps || !h->plan.full || h->plan.fmt != ARS_F32 || phase < 0 || phase >= h->plan.n_phases || len < (size_t) h->plan.n_taps)
    return B200_ERR_INVALID_ARG;
  memcpy (taps, &h->plan.phases[(size_t) phase * h->plan.n_taps], sizeof (float) * h->plan.n_taps);
  return h->plan.n_taps;
}


int b200_ars_process_host_submit (b200_ars * h, const void *in_host, size_t in_frames, void *out_host,
    size_t out_capacity_frames, size_t * out_frames)
{
  if (!h || (!out_host && out_capacity_frames)) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  B200_CUDA_TRY (h->ring.setup ());
  const size_t bpf = (size_t) h->plan.channels * h->plan.width;     // the caller's samples
  const size_t in_bytes = in_host ? in_frames * bpf : 0;
  const size_t want = b200_ars_get_out_frames (h, in_frames);
  if (want > out_capacity_frames) return B200_ERR_INVALID_ARG;
  const size_t out_bytes = want * bpf;
  auto & r = h->ring;
  B200_CUDA_TRY (r.take (in_bytes, in_bytes + in_bytes / 4, out_bytes, out_bytes + out_bytes / 4));
  if (in_bytes) B200_CUDA_TRY (r.upload (r.in (), in_host, in_bytes));
  B200_CUDA_TRY (r.inputs_ready ());
  size_t got = 0;
  int st = b200_ars_process (h, in_host ? r.in () : nullptr, in_frames, r.out (), want, &got, r.run_stream ());
  if (st != B200_OK) return st;
  B200_CUDA_TRY (r.run_done ());
  // the bytes the kernels wrote: the 20-bit _32 formats leave the last quarter of the caller's frames as it was
  const size_t written = (size_t) h->plan.channels * (h->plan.io.kind != ARS_IO_NONE ? h->plan.io.step : h->plan.width);
  if (got) B200_CUDA_TRY (r.download (out_host, r.out (), got * written));
  B200_CUDA_TRY (r.finish ());
  if (out_frames) *out_frames = got;
  return B200_OK;
}

int b200_ars_process_host_wait (b200_ars * h, int keep_in_flight)
{
  if (!h || keep_in_flight < 0 || keep_in_flight >= b200_ars::kSlots) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  if (h->ring.idle (keep_in_flight)) return B200_OK;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  B200_CUDA_TRY (h->ring.wait (keep_in_flight));
  return B200_OK;
}

int b200_ars_process_host (b200_ars * h, const void *in_host, size_t in_frames, void *out_host,
    size_t out_capacity_frames, size_t * out_frames)
{
  int st = b200_ars_process_host_submit (h, in_host, in_frames, out_host, out_capacity_frames, out_frames);
  if (st != B200_OK) return st;
  return b200_ars_process_host_wait (h, 0);
}

}  // extern "C"
