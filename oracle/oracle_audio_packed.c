/* oracle/oracle_audio_packed.c — TEST INFRASTRUCTURE ONLY.
 *
 * audioresample on the sample formats it does not hand to its resampler unconverted: the converter's generic path
 * (converter_generic, gst-libs/gst/audio/audio-converter.c:1281-1310) in plain C around the oracle resampler of
 * oracle_audio.c, which stays as it is:
 *   1. unpack to S32 (integer formats) or F64 (F32BE, F64BE) with GST_AUDIO_PACK_FLAG_TRUNCATE_RANGE (do_unpack :455-490);
 *      no input (drain) is silence of the unpack format, zeros
 *   2. resample in the unpack format
 *   3. quantize integer formats narrower than 32 bits (chain_quantize :968-1021, no dither, no noise shaping):
 *      audio_orc_int_bias, a saturating add of half a step and the bits below the depth cleared
 *   4. pack with flags 0 (:1305)
 * Unpack and pack per format: audio-format.c:116-217 and the ORC programs of gstaudiopack.orc.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

typedef struct {
  int format, width, step, depth, is_signed, big, is_float;
} PackedFormat;

/* GstAudioFormat value, bytes per sample in the buffer, bytes from one sample to the next (the 20-bit _32 formats use
 * the 3-byte pack functions, audio-format.c:206-213), depth, signed, big-endian, float */
static const PackedFormat kFormats[] = {
  {2, 1, 1, 8, 1, 0, 0}, {3, 1, 1, 8, 0, 0, 0},
  {5, 2, 2, 16, 1, 1, 0}, {6, 2, 2, 16, 0, 0, 0}, {7, 2, 2, 16, 0, 1, 0},
  {8, 4, 4, 24, 1, 0, 0}, {9, 4, 4, 24, 1, 1, 0}, {10, 4, 4, 24, 0, 0, 0}, {11, 4, 4, 24, 0, 1, 0},
  {13, 4, 4, 32, 1, 1, 0}, {14, 4, 4, 32, 0, 0, 0}, {15, 4, 4, 32, 0, 1, 0},
  {16, 3, 3, 24, 1, 0, 0}, {17, 3, 3, 24, 1, 1, 0}, {18, 3, 3, 24, 0, 0, 0}, {19, 3, 3, 24, 0, 1, 0},
  {20, 3, 3, 20, 1, 0, 0}, {21, 3, 3, 20, 1, 1, 0}, {22, 3, 3, 20, 0, 0, 0}, {23, 3, 3, 20, 0, 1, 0},
  {24, 3, 3, 18, 1, 0, 0}, {25, 3, 3, 18, 1, 1, 0}, {26, 3, 3, 18, 0, 0, 0}, {27, 3, 3, 18, 0, 1, 0},
  {29, 4, 4, 32, 1, 1, 1}, {31, 8, 8, 64, 1, 1, 1},
  {32, 4, 3, 20, 1, 0, 0}, {33, 4, 3, 20, 1, 1, 0}, {34, 4, 3, 20, 0, 0, 0}, {35, 4, 3, 20, 0, 1, 0},
};

typedef struct {
  OracleArs *r;
  PackedFormat f;
  int channels;
} OracleArsPacked;

OracleArsPacked *oracle_ars_new_packed (int in_rate, int out_rate, int channels, int quality, int format, int method,
    int filter_mode, int interpolation);
OracleArs *oracle_ars_packed_resampler (OracleArsPacked * p);
size_t oracle_ars_process_packed (OracleArsPacked * p, const void *in, size_t in_frames, void *out, size_t out_capacity);
void oracle_ars_free_packed (OracleArsPacked * p);
int oracle_ars_packed_width (int format);

static const PackedFormat *
find_format (int format)
{
  for (size_t i = 0; i < sizeof (kFormats) / sizeof (kFormats[0]); i++)
    if (kFormats[i].format == format)
      return &kFormats[i];
  return NULL;
}

/* bytes in the buffer of one sample of a packed format; 0 for the formats resampled unconverted and unknown ones */
int
oracle_ars_packed_width (int format)
{
  const PackedFormat *f = find_format (format);
  return f ? f->width : 0;
}

/* method / filter_mode / interpolation: the ORACLE_ARS_* values of oracle_ars_new_opts */
OracleArsPacked *
oracle_ars_new_packed (int in_rate, int out_rate, int channels, int quality, int format, int method, int filter_mode,
    int interpolation)
{
  const PackedFormat *f = find_format (format);
  OracleArsPacked *p;
  if (!f)
    return NULL;
  p = calloc (1, sizeof (*p));
  p->f = *f;
  p->channels = channels;
  p->r = oracle_ars_new_opts (in_rate, out_rate, channels, quality, f->is_float ? ORACLE_AFMT_F64 : ORACLE_AFMT_S32,
      method, filter_mode, interpolation);
  if (!p->r) {
    free (p);
    return NULL;
  }
  return p;
}

/* for update / reset / get_out_frames: the resampler works in the unpack format */
OracleArs *
oracle_ars_packed_resampler (OracleArsPacked * p)
{
  return p->r;
}

void
oracle_ars_free_packed (OracleArsPacked * p)
{
  if (!p)
    return;
  oracle_ars_free (p->r);
  free (p);
}

static uint64_t
read_sample (const PackedFormat * f, const uint8_t * s)
{
  uint64_t x = 0;
  for (int b = 0; b < f->step; b++)
    x |= (uint64_t) s[b] << (8 * (f->big ? f->step - 1 - b : b));
  return x;
}

static void
write_sample (const PackedFormat * f, uint8_t * d, uint64_t x)
{
  for (int b = 0; b < f->step; b++)
    d[b] = (uint8_t) (x >> (8 * (f->big ? f->step - 1 - b : b)));
}

/* ORC_DENORMAL / ORC_DENORMAL_DOUBLE of convfd / convdf */
static uint32_t
flush32 (uint32_t b)
{
  return (b & 0x7f800000u) ? b : (b & 0xff800000u);
}

static uint64_t
flush64 (uint64_t b)
{
  return (b & 0x7ff0000000000000ull) ? b : (b & 0xfff0000000000000ull);
}

static void
unpack (const PackedFormat * f, const uint8_t * in, void *tmp, size_t n)
{
  for (size_t i = 0; i < n; i++) {
    const uint64_t x = read_sample (f, in + i * f->step);
    if (!f->is_float) {
      /* the _trunc programs and MAKE_PACK_UNPACK: the sample moved to the top of 32 bits, sign bit flipped if unsigned */
      ((int32_t *) tmp)[i] = (int32_t) (((uint32_t) x << (32 - f->depth)) ^ (f->is_signed ? 0u : 0x80000000u));
    } else if (f->width == 4) {
      const uint32_t b = flush32 ((uint32_t) x);
      float v;
      memcpy (&v, &b, 4);
      ((double *) tmp)[i] = v;
    } else
      memcpy ((double *) tmp + i, &x, 8);
  }
}

static void
quantize_pack (const PackedFormat * f, void *tmp, uint8_t * out, size_t n)
{
  const int shift = 32 - f->depth;
  for (size_t i = 0; i < n; i++) {
    uint8_t *d = out + i * f->step;
    if (!f->is_float) {
      int32_t v = ((int32_t *) tmp)[i];
      uint32_t u;
      if (shift) {
        int64_t t = (int64_t) v + ((int64_t) 1 << (shift - 1));
        if (t > INT32_MAX)
          t = INT32_MAX;
        v = (int32_t) ((uint32_t) t & ~((1u << shift) - 1));
      }
      u = (uint32_t) v ^ (f->is_signed ? 0u : 0x80000000u);
      /* pack_s24_32 / _s32 shift arithmetically (shrsl); the others logically or keep only the bits they write */
      write_sample (f, d, (f->is_signed && f->step == 4) ? (uint32_t) ((int32_t) u >> shift) : u >> shift);
    } else if (f->width == 4) {
      uint64_t b;
      uint32_t fb;
      double v;
      float s;
      memcpy (&b, (double *) tmp + i, 8);
      b = flush64 (b);
      memcpy (&v, &b, 8);
      s = (float) v;
      memcpy (&fb, &s, 4);
      write_sample (f, d, flush32 (fb));
    } else {
      uint64_t b;
      memcpy (&b, (double *) tmp + i, 8);
      write_sample (f, d, b);
    }
  }
}

/* like oracle_ars_process_any: in == NULL pushes silence; writes the frames the resampler produces as packed samples,
 * nothing past them (the 20-bit _32 formats leave the last quarter of the frames' bytes untouched) */
size_t
oracle_ars_process_packed (OracleArsPacked * p, const void *in, size_t in_frames, void *out, size_t out_capacity)
{
  const size_t bps = p->f.is_float ? 8 : 4, ch = (size_t) p->channels;
  void *tin = calloc (in_frames * ch + 1, bps), *tout = calloc (out_capacity * ch + 1, bps);
  size_t n;
  if (in)
    unpack (&p->f, in, tin, in_frames * ch);
  n = oracle_ars_process_any (p->r, tin, in_frames, tout, out_capacity);
  quantize_pack (&p->f, tout, out, n * ch);
  free (tin);
  free (tout);
  return n;
}
