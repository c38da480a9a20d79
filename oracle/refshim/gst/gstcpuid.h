/* refshim: <gst/gstcpuid.h> — report the SSE levels every x86-64 host has, so the
 * reference picks the same SSE inner products its real x86 build uses
 * (gst-libs/gst/audio/audio-resampler-x86.h:29-70). */
#ifndef B200_REFSHIM_CPUID_H
#define B200_REFSHIM_CPUID_H
#include <gst/gst.h>
static inline gboolean gst_cpuid_supports_x86_sse2 (void) { return __builtin_cpu_supports ("sse2"); }
static inline gboolean gst_cpuid_supports_x86_sse4_1 (void) { return __builtin_cpu_supports ("sse4.1"); }
#endif
