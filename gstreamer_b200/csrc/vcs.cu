// gstreamer_b200/csrc/vcs.cu — b200_vcs_* entry points (product code).
//
// Replaces gst_video_converter_new/_frame/_free for the element's transform_frame()
// (gst-plugins-base/gst/videoconvertscale/gstvideoconvertscale.c:1981-2005); device
// calling convention after gst_cuda_converter_convert_frame
// (gst-plugins-bad/gst-libs/gst/cuda/gstcudaconverter.cpp:1911).
#include "common.h"
#include "vcs_plan.h"
#include "video_format.h"
#include "vcs_device.h"
#include "vcs_kernels.cuh"
#include "vcs_lanczos2.cuh"
#include "vcs_lanczos2_v2.cuh"
#include "vcs_l2mma.cuh"
#ifndef B200_CUDA_EMU
#include "vcs_l2tc.cuh"          // wgmma: no host emulation
#endif
#include "vcs_light.cuh"
#include "vcs_ntap.cuh"
#include "vcs_planes.cuh"
#include "vcs_down420.cuh"
#include "vcs_rgb420.cuh"
#include "vcs_yuy2_420.cuh"

#include <string.h>
#include <algorithm>
#include <new>
#include <vector>

using namespace b200;

// A/B and tuning switches of the converter (DESIGN.md §4.3b), read once when a handle is created
struct VcsKnobs {
  bool cross_generic = false;     // B200_CROSS_GENERIC: the 4:2:0 -> other 4:2:0 chain runs the generic kernel
  bool rgb420_generic = false;    // B200_RGB420_GENERIC: packed RGB / 4:2:2 -> 4:2:0 runs the chain
  bool l2_v1 = false;             // B200_L2_V1: no second form of the 2:1 kernel
  bool l2_x4 = false;             // B200_L2_X4 (any value): no second form where it is the only form
  bool l2_tc = false;             // B200_L2_TC=1: the tensor-core 2:1 kernel (variant 7) by default
  bool planes_slow = false;       // B200_PLANES_SLOW: the byte-wise plane kernel for every plane
};

struct b200_vcs {
  VcsPlan plan;
  int device = -1;
  VcsKnobs knobs;
  VcsDev dev;                     // kernel parameter block (device pointers inside)
  int variant = 0;                // the kernel the handle asks for (default or b200_vcs_set_kernel_variant)
  // device tables
  uint32_t *d_hoff = nullptr, *d_voff = nullptr;
  int16_t *d_hcoef = nullptr, *d_vcoef = nullptr, *d_hsum = nullptr, *d_vsum = nullptr;
  uint8_t *d_cmode = nullptr;
  // host<->device pipeline for system-memory peers
  static const int kSlots = 4, kChunk = 4;
  uint8_t *slot_in[kSlots] = {nullptr}, *slot_out[kSlots] = {nullptr};
  cudaStream_t s_h2d = nullptr, s_run = nullptr, s_d2h = nullptr;
  cudaEvent_t ev_in[kSlots] = {nullptr}, ev_run[kSlots] = {nullptr}, ev_out[kSlots] = {nullptr};
  bool pipeline_ready = false;
  int slot_frames = 0;            // frames each slot holds (one kernel launch per slot-full)
  Lanczos2Tables l2_tables;
  Lanczos2State l2;
  Lanczos2V2Tables l2v2_tables;      // second form of the headline kernel (vcs_lanczos2_v2.cuh) where the plan allows it
  Lanczos2V2State l2v2;
  NtapState ntap;
  L2mmaTables mma_tables;         // experimental tensor-path variant of the 2:1 kernel (variant 6, opt-in)
  L2mmaState mma;
#ifndef B200_CUDA_EMU
  L2tcTables tc_tables;           // tensor-core (wgmma) formulation of the 2:1 kernel (variant 7)
  L2tcState tc;
#endif
  PlanesState planes;
  // 4:2:0 -> other 4:2:0 family: scaled A,Y,U,V scratch images between the two launches
  Down420Dev down;
  BorderDev border;               // destination rectangle: what to fill around it
  uint8_t *d_scratch = nullptr;
  int scratch_frames = 0;
  size_t scratch_frame_bytes = 0;
  // packed RGB -> 4:2:0 at an unchanged or shrinking size: [word-wide scaler on 4-byte pixels ->] matrix + down-sample + pack
  Rgb420Dev rgb420;
  Rgb2AyuvDev rgb2ayuv;           // the frame grows: the matrix runs first, on its own
  Yuy2AyuvDev yuy2ayuv;           // packed 4:2:2 input: unpack + horizontal chroma up-sampling, on its own
  bool rgb420_ok = false, rgb420_scaled = false;
  int rgb420_pre = 0;             // 0: none, 1: vcs_rgb2ayuv_kernel, 2: vcs_yuy2_ayuv_kernel
  PlaneFastState rgb420_scaler;
  Yuy2Dev yuy2;                   // YUY2 / UYVY -> I420 / YV12 at an unchanged size (plan.yuy2_420)
  DeintDev deint;                 // packed RGB -> RGBP / BGRP: the de-interleave (after planes' scaler into d_scratch if scaled)
  bool deint_scaled = false;
  size_t in_bytes = 0, out_bytes = 0;
};

namespace {

VcsKnobs read_knobs ()
{
  VcsKnobs k;
  k.cross_generic = getenv ("B200_CROSS_GENERIC") != nullptr;
  k.rgb420_generic = getenv ("B200_RGB420_GENERIC") != nullptr;
  k.l2_v1 = getenv ("B200_L2_V1") != nullptr;
  k.l2_x4 = getenv ("B200_L2_X4") != nullptr;
  const char *tc = getenv ("B200_L2_TC");
  k.l2_tc = tc && tc[0] == '1';
  k.planes_slow = getenv ("B200_PLANES_SLOW") != nullptr;
  return k;
}

// the largest power of two up to 16 that divides every frame pointer of a batch
template <typename T> int alignment (T *const *frames, int n)
{
  uintptr_t bits = 16;
  for (int i = 0; i < n; i++) bits |= (uintptr_t) frames[i];
  return (int) (bits & (~bits + 1));
}

// the handle's scratch image: `bytes` per frame for n frames
int ensure_scratch (b200_vcs * h, size_t bytes, int n)
{
  if (n <= h->scratch_frames && bytes == h->scratch_frame_bytes) return B200_OK;
  B200_CUDA_TRY (cudaFree (h->d_scratch));                          // synchronises with launches still reading it
  h->d_scratch = nullptr; h->scratch_frames = 0;
  B200_CUDA_TRY (cudaMalloc ((void **) &h->d_scratch, bytes * n));
  h->scratch_frames = n; h->scratch_frame_bytes = bytes;
  return B200_OK;
}

// What one convert launches after the border fill.  Path::one is a single kernel (Kern); Path::chain is Kern into the
// scratch image, [the generic kernel for the extra row,] vcs_down420_kernel.
enum class Path { planes, deint, yuy2, rgb420, chain, one };
enum Kern { K_GENERIC, K_L2, K_L2V2, K_LIGHT, K_NTAP, K_MMA, K_TC };
const int kern_variant[] = {0, 1, 1, 2, 3, 6, 7};
const char *const kern_name[] = {"vcs_generic_kernel", "vcs_lanczos2_kernel", "vcs_lanczos2_v2_kernel", "vcs_light_kernel",
                                 "vcs_ntap_kernel", "vcs_l2mma_kernel", "vcs_l2tc_kernel"};

struct Route {
  int status = B200_OK;           // B200_ERR_INVALID_ARG: packed RGB input that is not word aligned
  Path path = Path::one;
  Kern kern = K_GENERIC;
  bool planes_aligned = false;    // Path::planes / deint: the planes' word-wide launches may run (8-byte aligned frames)
  int kernel_variant = 0;         // b200_vcs_plan_info.kernel_variant
  const char *name = "";          // b200_vcs_kernel_name
  int named_variant = 0;          // Path::one / chain: the variant whose kernel `name` is (0: the generic one)
  int n_launches = 0;             // b200_vcs_plan_info.n_launches_per_convert, the border fill included
};

// The one place that decides which kernels a convert launches: from the plan, the prepared states, the kernel variant
// asked for and the alignment of the batch's in / out frames (ain, aout: see alignment ()).  Introspection passes 16.
// A host-only handle prepares nothing; it reports what the plan selects, with the first form of the 2:1 kernel in
// place of the second.
Route select_route (const b200_vcs * h, int variant, int ain, int aout)
{
  const VcsPlan & p = h->plan;
  const bool host = h->device < 0;
  const int border = p.has_dest && p.fill_border ? 1 : 0;
  Route r;
  if (p.planes_mode) {
    r.kernel_variant = 4;
    if (p.rgbp_out) {                                               // [the packed RGB scaler into the scratch image ->] de-interleave
      r.path = Path::deint;
      r.planes_aligned = ain >= 8;
      r.name = "vcs_rgb_deinterleave_kernel";
      r.n_launches = border + 1 + (h->deint_scaled ? plane_launches (h->planes, r.planes_aligned) : 0);
    } else {
      r.path = Path::planes;
      r.planes_aligned = ain >= 8 && aout >= 8;
      r.name = planes_kernel_name (h->planes);
      r.n_launches = border + plane_launches (h->planes, r.planes_aligned);
    }
    return r;
  }
#ifndef B200_CUDA_EMU
  const bool tc_ready = h->tc.ready;
#else
  const bool tc_ready = false;                                    // wgmma: no host emulation
#endif
  const bool l2v2 = h->l2v2.ready && h->l2.x4;
  const bool l2_first = !p.planar && !p.rgbp_out;                 // what the first form of the 2:1 kernel reads and writes
  const bool ntap_ready = h->ntap.ready || host;
  if (!p.yuv_out) {
    if (variant == 6 && h->mma.ready && ain >= 8 && aout >= 4) r.kern = K_MMA;             // 64-bit plane loads
    else if (variant == 7 && tc_ready && ain >= 16 && aout >= 4) r.kern = K_TC;             // 16-byte cp.async of the luma rows
    else if (variant == 7 && tc_ready && p.lanczos2_ok && l2_first) r.kern = K_L2;
    else if (variant == 1 && p.lanczos2_ok && (l2v2 || l2_first || host)) r.kern = l2v2 ? K_L2V2 : K_L2;
    else if (variant == 2 && p.light_ok && ain >= 4) r.kern = K_LIGHT;                      // 32-bit plane loads
    else if (variant == 3 && p.ntap_ok && ntap_ready && ain >= 4) r.kern = K_NTAP;
  }
  if (r.kern == K_GENERIC && p.rgb_in && ain < 4) r.status = B200_ERR_INVALID_ARG;           // packed pixels: 32-bit loads
  if (r.kern != K_GENERIC || !p.yuv_out) {
    r.path = Path::one;
    r.n_launches = 1;
  } else if (p.yuy2_420) {
    r.path = Path::yuy2;
    r.name = "vcs_yuy2_420_kernel";
    r.n_launches = 1;
  } else if (h->rgb420_ok && (h->rgb420_pre != 2 || ain >= 4)) {     // vcs_yuy2_ayuv_kernel reads pixel pairs as words
    r.path = Path::rgb420;
    r.name = h->rgb420_pre == 2 ? "vcs_yuy2_ayuv_kernel" : "vcs_rgb420_kernel";
    r.n_launches = 1 + (h->rgb420_pre ? 1 : 0) + (h->rgb420_scaled ? 1 : 0);
  } else {
    // the chain up to the scaled pixels: the 2:1 / light / n-tap kernels (matrix stage off) where the plan allows, else
    // the generic one
    r.path = Path::chain;
    if (variant == 1 && p.lanczos2_ok && ((l2v2 && ain >= 8) || host)) r.kern = l2v2 ? K_L2V2 : K_L2;
    else if (variant == 2 && p.light_ok && ain >= 4) r.kern = K_LIGHT;
    else if (variant == 3 && p.ntap_ok && ntap_ready && ain >= 4) r.kern = K_NTAP;
    r.n_launches = p.extra_row ? 3 : 2;
  }
  if (r.path == Path::one || r.path == Path::chain) {
    r.name = kern_name[r.kern];
    r.named_variant = kern_variant[r.kern];
    // B200_CROSS_GENERIC swaps the chain's first launch only: the handle still names the kernel of its variant
    if (r.path == Path::chain && h->knobs.cross_generic) r.kern = K_GENERIC;
  }
  r.kernel_variant = p.yuv_out ? 5 : r.named_variant;
  r.n_launches += border;
  return r;
}

// the variant a new handle runs: the first of 7 (B200_L2_TC=1), 1, 2, 3 whose kernel the route names, else 0
int default_variant (const b200_vcs * h)
{
  for (int v : {7, 1, 2, 3})
    if ((v != 7 || h->knobs.l2_tc) && select_route (h, v, 16, 16).named_variant == v) return v;
  return 0;
}

int upload_axis (const AxisPlan & a, uint32_t **off, int16_t **coef, int16_t **sum, AxisDev * d)
{
  int st;
  if ((st = upload (off, a.offset.data (), a.offset.size ())) != B200_OK) return st;
  if ((st = upload (coef, a.coef.data (), a.coef.size ())) != B200_OK) return st;
  if ((st = upload (sum, a.sum.data (), a.sum.size ())) != B200_OK) return st;
  d->offset = *off; d->coef = *coef; d->sum = *sum;
  d->mode = a.mode; d->n_taps = a.n_taps; d->coef_per_out = a.coef_per_out; d->span = a.span;
  d->out_size = a.out_size; d->in_size = a.in_size;
  return B200_OK;
}

// packed RGB -> 4:2:0 with every scaler in front of the matrix (the frame does not grow) and no destination rectangle:
// vcs_rgb420.cuh.  Leaves rgb420_ok false (the generic chain runs) for what the fast kernels decline.
int prepare_rgb420 (b200_vcs * h)
{
  const VcsPlan & p = h->plan;
  h->rgb420_ok = false;
  const bool packed422 = p.in_422_444 && p.ystep == 2;            // YUY2 / UYVY / YVYU
  if (!(p.rgb_in || packed422) || !p.yuv_out || p.yuy2_420 || h->knobs.rgb420_generic) return B200_OK;
  Rgb420Dev & r = h->rgb420;
  memset (&r, 0, sizeof (r));
  if (p.rgb_in) {
    const int pos_r = p.in_sel & 0xf, pos_g = (p.in_sel >> 4) & 0xf, pos_b = (p.in_sel >> 8) & 0xf;
    for (int i = 0; i < 3; i++) {
      if (!rgb420_split_row (p.m_rgb2yuv[i], pos_r, pos_g, pos_b, &r.ca[i], &r.cb[i])) return B200_OK;
      r.off[i] = p.m_rgb2yuv[i][3];
    }
  } else if ((p.in.stride[0] & 3) || (p.in.offset[0] & 3)) return B200_OK;      // pixel pairs are read as words
  const Down420Dev & q = h->down;
  r.ow = q.ow; r.oh = q.oh; r.hmode = q.hmode; r.vavg = q.vavg;
  r.stride_y = q.stride_y; r.stride_u = q.stride_u; r.stride_v = q.stride_v; r.cstep = q.cstep;
  r.off_y = q.off_y; r.off_u = q.off_u; r.off_v = q.off_v;
  const unsigned long long cbase = q.cstep == 2 ? std::min (q.off_u, q.off_v) : (q.off_u | q.off_v);
  r.wvec = ((q.stride_y | q.stride_u | q.stride_v) & 3) == 0 && ((q.off_y | cbase) & 3) == 0;
  h->rgb420_scaled = p.h.scaling || p.v.scaling;
  // a kernel of its own in front of the scalers: the RGB -> YUV matrix when the frame grows (chain_scale puts the
  // scalers behind it), unpack + horizontal chroma up-sampling for packed 4:2:2
  h->rgb420_pre = packed422 ? 2 : (p.matrix_first && h->rgb420_scaled) ? 1 : 0;
  int in_stride = p.in.stride[0];
  unsigned long long in_off = p.in.offset[0];
  if (h->rgb420_pre) {
    const int dstride = (p.in.width * 4 + 15) & ~15;
    if (h->rgb420_pre == 1) {
      Rgb2AyuvDev & m = h->rgb2ayuv;
      memset (&m, 0, sizeof (m));
      m.w = p.in.width; m.h = p.in.height; m.sstride = p.in.stride[0]; m.soff = p.in.offset[0]; m.dstride = dstride;
      for (int i = 0; i < 3; i++) { m.ca[i] = r.ca[i]; m.cb[i] = r.cb[i]; m.off[i] = r.off[i]; }
    } else {
      Yuy2AyuvDev & m = h->yuy2ayuv;
      memset (&m, 0, sizeof (m));
      m.w = p.in.width; m.h = p.in.height; m.sstride = p.in.stride[0]; m.soff = p.in.offset[0]; m.dstride = dstride;
      // byte positions inside a pixel-pair word, from the plan's sample offsets (YUY2: Y0 U Y1 V; UYVY: U Y0 V Y1; YVYU: Y0 V Y1 U)
      m.ypos = (int) (p.in_off_y - p.in.offset[0]); m.upos = (int) (p.in_off_u - p.in.offset[0]); m.vpos = (int) (p.in_off_v - p.in.offset[0]);
      m.cosited = p.h_cosited ? 1 : 0;
    }
    in_stride = dstride; in_off = 0;
  }
  if (!h->rgb420_scaled) {
    r.sstride = in_stride; r.soff = in_off;
    r.svec = (r.sstride & 15) == 0 && (r.soff & 15) == 0;
  } else {
    PlanePlan pl;
    pl.src_plane = 0; pl.iw = p.in.width; pl.ih = p.in.height; pl.ow = p.out.width; pl.oh = p.out.height;
    pl.ne = 4; pl.swz = 0; pl.mode = PM_SCALE;
    pl.have_h = p.h.scaling; pl.have_v = p.v.scaling; pl.h_first = p.h_first;
    pl.h = p.h; pl.v = p.v;
    const int sstride = (p.out.width * 4 + 15) & ~15;
    std::vector<int32_t> hp, vp;
    if (!plan_plane_fast (pl, in_stride, in_off, sstride, 0, &h->rgb420_scaler, &hp, &vp)) return B200_OK;
    const int st = prepare_plane_fast (pl, hp, vp, &h->rgb420_scaler);
    if (st != B200_OK) return st;
    r.sstride = sstride; r.soff = 0; r.svec = 1;
  }
  h->rgb420_ok = true;
  return B200_OK;
}

// one launch of kernel k: the single kernel of Path::one, the chain's first launch (into the scratch image)
int launch_kern (b200_vcs * h, Kern k, const VcsBatch & batch, int n, cudaStream_t stream)
{
  const VcsPlan & p = h->plan;
  switch (k) {
    case K_L2: return launch_lanczos2 (h->dev, h->l2, batch, n, stream);
    case K_L2V2: return launch_lanczos2_v2 (h->dev, h->l2, h->l2v2, batch, n, stream, p.rgbp_out);
    case K_LIGHT: return launch_light (h->dev, p, batch, n, stream);
    case K_NTAP: return launch_ntap (h->dev, p, h->ntap, batch, n, stream);
    case K_MMA: return launch_l2mma (h->dev, h->mma, batch, n, stream);
#ifndef B200_CUDA_EMU
    case K_TC: return launch_l2tc (h->dev, h->tc, batch, n, stream);
#endif
    default: break;
  }
  dim3 grid ((p.out.width + p.tile_w - 1) / p.tile_w, (p.out.height + p.tile_h - 1) / p.tile_h, n);
  if (p.rgbp_out) vcs_generic_kernel<true> <<<grid, 256, p.smem_bytes, stream>>> (h->dev, batch);
  else vcs_generic_kernel<false> <<<grid, 256, p.smem_bytes, stream>>> (h->dev, batch);
  B200_CUDA_TRY (cudaGetLastError ());
  return B200_OK;
}

int launch_convert (b200_vcs * h, int n, const VcsBatch & batch, cudaStream_t stream)
{
  const VcsPlan & p = h->plan;
  const int ain = alignment (batch.in, n), aout = alignment (batch.out, n);
  const Route r = select_route (h, h->variant, ain, aout);
  int st;
  if (p.has_dest && p.fill_border) {
    // border and rectangle are disjoint byte sets: the fill simply goes first on the same stream
    BorderBatch b;
    int wmax = 0, hmax = 0;
    for (int i = 0; i < n; i++) b.out[i] = batch.out[i];
    for (int i = 0; i < h->border.n_planes; i++) {
      wmax = max (wmax, h->border.pl[i].pw); hmax = max (hmax, h->border.pl[i].ph);
    }
    dim3 grid ((wmax + 255) / 256, hmax, h->border.n_planes * n);
    vcs_border_kernel <<<grid, 256, 0, stream>>> (h->border, b);
    B200_CUDA_TRY (cudaGetLastError ());
  }
  if (r.status != B200_OK) return r.status;
  switch (r.path) {
    case Path::planes:
      return launch_planes (h->planes, batch, n, stream, r.planes_aligned);
    case Path::deint: {
      // packed RGB -> RGBP / BGRP: [the packed RGB scaler into the scratch image ->] de-interleave
      DeintBatch fin;
      for (int i = 0; i < n; i++) { fin.src[i] = batch.in[i]; fin.out[i] = batch.out[i]; }
      if (h->deint_scaled) {
        const size_t frame = (size_t) h->deint.sstride * h->deint.h;
        if ((st = ensure_scratch (h, frame, n)) != B200_OK) return st;
        VcsBatch mid;
        for (int i = 0; i < n; i++) { mid.in[i] = batch.in[i]; mid.out[i] = h->d_scratch + frame * i; fin.src[i] = mid.out[i]; }
        if ((st = launch_planes (h->planes, mid, n, stream, r.planes_aligned)) != B200_OK) return st;
      }
      return launch_rgb_deinterleave (h->deint, fin, n, stream);
    }
    case Path::yuy2: {
      Yuy2Dev y = h->yuy2;
      Yuy2Batch b;
      for (int i = 0; i < n; i++) { b.src[i] = batch.in[i]; b.out[i] = batch.out[i]; }
      if (ain < 16 && y.svec > 1) y.svec = 1;
      if (ain < 4) y.svec = 0;
      if (aout < 4) y.wvec = 0;
      return launch_yuy2_420 (y, b, n, stream);
    }
    case Path::rgb420: {
      // [vcs_rgb2ayuv_kernel / vcs_yuy2_ayuv_kernel ->] [the word-wide scaler ->] matrix + down-sample + pack
      Rgb420Dev rd = h->rgb420;
      if (aout < 4) rd.wvec = 0;
      const int pre = h->rgb420_pre;
      const int pre_stride = pre == 1 ? h->rgb2ayuv.dstride : pre == 2 ? h->yuy2ayuv.dstride : 0;
      const size_t pre_bytes = (size_t) pre_stride * p.in.height;
      const size_t scaled_bytes = h->rgb420_scaled ? (size_t) rd.sstride * p.out.height : 0;
      const size_t frame = pre_bytes + scaled_bytes;
      if (frame && (st = ensure_scratch (h, frame, n)) != B200_OK) return st;
      VcsBatch mid;                                                 // the scaler's view: in = the pre kernel's image or the frame
      Rgb420Batch fin;
      for (int i = 0; i < n; i++) { mid.in[i] = batch.in[i]; fin.out[i] = batch.out[i]; }
      if (pre) {
        Rgb420Batch pre_b;
        for (int i = 0; i < n; i++) { pre_b.src[i] = batch.in[i]; pre_b.out[i] = h->d_scratch + frame * i + scaled_bytes; mid.in[i] = pre_b.out[i]; }
        st = pre == 1 ? launch_rgb2ayuv (h->rgb2ayuv, pre_b, n, stream) : launch_yuy2_ayuv (h->yuy2ayuv, pre_b, n, stream);
        if (st != B200_OK) return st;
      }
      if (h->rgb420_scaled) {
        for (int i = 0; i < n; i++) { mid.out[i] = h->d_scratch + frame * i; fin.src[i] = mid.out[i]; }
        if ((st = launch_plane_fast (h->rgb420_scaler, mid, n, stream)) != B200_OK) return st;
      } else {
        for (int i = 0; i < n; i++) fin.src[i] = mid.in[i];
        if (alignment (mid.in, n) < 16) rd.svec = 0;
      }
      return launch_rgb420 (rd, fin, n, stream, pre == 0);
    }
    case Path::chain: {
      // launch 1 writes the scaled pixels of every frame to its scratch image, launch 2 down-samples and packs
      const size_t frame = (size_t) h->down.stride_s * (p.out.height + (p.extra_row ? 1 : 0));
      if ((st = ensure_scratch (h, frame, n)) != B200_OK) return st;
      VcsBatch mid;
      Down420Batch fin;
      for (int i = 0; i < n; i++) {
        mid.in[i] = batch.in[i]; mid.out[i] = h->d_scratch + frame * i;
        fin.scratch[i] = mid.out[i]; fin.out[i] = batch.out[i];
      }
      if ((st = launch_kern (h, r.kern, mid, n, stream)) != B200_OK) return st;
      if (p.extra_row) {
        // scratch row `oh`: the chain over a one-line view of the frame (its last line, chroma row unfiltered vertically)
        VcsDev x = h->dev;
        x.off_y += (unsigned long long) (p.in.height - 1) * x.stride_y;
        x.off_u += (unsigned long long) ((p.in.height - 1) >> 1) * x.stride_u;
        x.off_v += (unsigned long long) ((p.in.height - 1) >> 1) * x.stride_v;
        x.ih = 1; x.oh = 1; x.v.in_size = x.v.out_size = 1;
        x.off_out = (unsigned long long) p.out.height * x.stride_out;
        dim3 gx ((p.out.width + p.tile_w - 1) / p.tile_w, 1, n);
        vcs_generic_kernel<false> <<<gx, 256, p.smem_bytes, stream>>> (x, mid);
        B200_CUDA_TRY (cudaGetLastError ());
      }
      const int cw = (p.out.width + 1) / 2, chh = (p.out.height + 1) / 2;
      dim3 blk (32, 8), g2 ((cw + 31) / 32, (chh + 7) / 8, n);
      vcs_down420_kernel <<<g2, blk, 0, stream>>> (h->down, fin);
      B200_CUDA_TRY (cudaGetLastError ());
      return B200_OK;
    }
    case Path::one:
      break;
  }
  return launch_kern (h, r.kern, batch, n, stream);
}

// what a device handle uploads and derives for its launches (the handle's device is current)
int prepare_device (b200_vcs * h)
{
  const VcsPlan & p = h->plan;
  int st;
  if (p.planes_mode && p.rgbp_out) {
    // packed RGB -> planar RGB: the scaler writes a scratch image of 4-byte pixels (16-byte aligned rows), the
    // de-interleave reads it - or the input frame itself at an unchanged size
    DeintDev & d = h->deint;
    memset (&d, 0, sizeof (d));
    d.w = p.out.width; d.h = p.out.height; d.sel = p.deint_sel;
    for (int k = 0; k < 3; k++) { d.off[k] = p.out.offset[k]; d.stride[k] = p.out.stride[k]; }
    if (!h->deint_scaled) {
      d.soff = p.in.offset[0]; d.sstride = p.in.stride[0];
      return B200_OK;
    }
    VcsPlan sp = p;
    sp.out.offset[0] = 0; sp.out.stride[0] = (p.out.width * 4 + 15) & ~15;
    d.soff = 0; d.sstride = sp.out.stride[0];
    return prepare_planes (sp, &h->planes, h->knobs.planes_slow);
  }
  if (p.planes_mode) return prepare_planes (p, &h->planes, h->knobs.planes_slow);   // YUV -> same YUV family: plane scaling
  VcsDev & d = h->dev;
  memset (&d, 0, sizeof (d));
  d.iw = p.in.width; d.ih = p.in.height; d.ow = p.out.width; d.oh = p.out.height;
  d.stride_y = p.in.stride[0]; d.stride_c = p.in.stride[1]; d.stride_out = p.out.stride[0];
  d.off_y = p.in.offset[0]; d.off_c = p.in.offset[1]; d.off_out = p.out.offset[0];
  d.u_index = p.u_index; d.h_cosited = p.h_cosited; d.v_pairs = p.v_pairs;
  d.planar = p.planar ? 1 : 0; d.chroma_nearest = p.chroma_nearest ? 1 : 0;
  if (p.planar) {
    d.off_u = p.in.offset[p.plane_u]; d.off_v = p.in.offset[p.plane_v];
    d.stride_u = p.in.stride[p.plane_u]; d.stride_v = p.in.stride[p.plane_v];
  } else {                                                        // interleaved pairs: both components walk the same rows
    d.off_u = p.in.offset[1] + p.u_index; d.off_v = p.in.offset[1] + (p.u_index ^ 1);
    d.stride_u = d.stride_v = p.in.stride[1];
  }
  d.cstep = p.planar ? 1 : 2;
  d.ystep = 1; d.chshift = 1; d.cvshift = 1;
  if (p.in_422_444) {                                             // capture formats: explicit sample geometry
    d.off_y = p.in_off_y; d.off_u = p.in_off_u; d.off_v = p.in_off_v;
    d.stride_u = p.in_stride_u; d.stride_v = p.in_stride_v; d.cstep = p.cstep_in;
    d.ystep = p.ystep; d.chshift = p.chshift; d.cvshift = p.cvshift;
  }
  d.h_first = p.h_first; d.matrix_first = p.matrix_first;
  d.yuv_out = p.yuv_out ? 1 : 0;
  d.rgb_in = p.rgb_in ? 1 : 0; d.in_sel = p.in_sel;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 4; j++) d.m[i][j] = p.m_rgb2yuv[i][j];
  if (p.yuv_out) {                                                // the chain's output is the scratch image
    d.stride_out = p.out.width * 4; d.off_out = 0;
    Down420Dev & q = h->down;
    memset (&q, 0, sizeof (q));
    q.ow = p.out.width; q.oh = p.out.height; q.stride_s = d.stride_out;
    q.hmode = p.down_h; q.vavg = p.down_v ? 1 : 0; q.extra_row = p.extra_row ? 1 : 0;
    q.stride_y = p.out.stride[0]; q.off_y = p.out.offset[0];
    q.stride_u = p.out.stride[p.out_plane_u]; q.stride_v = p.out.stride[p.out_plane_v];
    q.cstep = p.out_cstep;
    q.off_u = p.out.offset[p.out_plane_u] + (p.out_cstep == 2 ? p.out_u_index : 0);
    q.off_v = p.out.offset[p.out_plane_v] + (p.out_cstep == 2 ? (p.out_u_index ^ 1) : 0);
    if ((st = prepare_rgb420 (h)) != B200_OK) return st;
    if (p.yuy2_420) {
      Yuy2Dev & y = h->yuy2;
      memset (&y, 0, sizeof (y));
      const bool y_odd = video_format (p.in.format)->pair_y == 1;   // UYVY: luma in the odd bytes
      y.w = p.in.width; y.h = p.in.height; y.sstride = p.in.stride[0]; y.soff = p.in.offset[0];
      y.sel_y = y_odd ? 0x7531 : 0x6420; y.sel_c = y_odd ? 0x6420 : 0x7531;
      y.svec = ((y.sstride | y.soff) & 15) == 0 ? 2 : (((y.sstride | y.soff) & 3) == 0 ? 1 : 0);
      y.stride_y = q.stride_y; y.stride_u = q.stride_u; y.stride_v = q.stride_v;
      y.off_y = q.off_y; y.off_u = q.off_u; y.off_v = q.off_v;
      y.wvec = ((q.stride_y | q.stride_u | q.stride_v) & 3) == 0 && ((q.off_y | q.off_u | q.off_v) & 3) == 0;
    }
  }
  d.p1 = p.p[0]; d.p2 = p.p[1]; d.p3 = p.p[2]; d.p4 = p.p[3]; d.p5 = p.p[4];
  d.sel = p.byte_sel[0] | (p.byte_sel[1] << 4) | (p.byte_sel[2] << 8) | (p.byte_sel[3] << 12);
  d.tile_w = p.tile_w; d.tile_h = p.tile_h; d.max_rows = p.max_rows; d.cols_pitch = p.cols_pitch;
  d.max_crows = p.max_crows;
  for (int k = 0; k < 3; k++) {                                   // planar RGB output planes (store_planar_px)
    d.off_pl[k] = p.rgbp_out ? p.out.offset[k] : 0; d.stride_pl[k] = p.rgbp_out ? p.out.stride[k] : 0;
  }
  if ((st = upload_axis (p.h, &h->d_hoff, &h->d_hcoef, &h->d_hsum, &d.h)) != B200_OK ||
      (st = upload_axis (p.v, &h->d_voff, &h->d_vcoef, &h->d_vsum, &d.v)) != B200_OK ||
      (st = upload (&h->d_cmode, p.chroma_mode.data (), p.chroma_mode.size ())) != B200_OK)
    return st;
  d.chroma_mode = h->d_cmode;
  if ((st = allow_max_dyn_smem (p.rgbp_out ? vcs_generic_kernel<true> : vcs_generic_kernel<false>)) != B200_OK) return st;
  if (h->mma_tables.ok && (st = prepare_l2mma (h->mma_tables, &h->mma)) != B200_OK) return st;
  if (p.lanczos2_ok) {
    if ((st = prepare_lanczos2 (h->l2_tables, h->dev, &h->l2)) != B200_OK) return st;
    if (h->l2v2_tables.ok && !h->knobs.l2_v1 && (st = prepare_lanczos2_v2 (h->l2v2_tables, &h->l2v2)) != B200_OK) return st;
#ifndef B200_CUDA_EMU
    if ((st = prepare_l2tc (h->tc_tables, &h->tc)) != B200_OK) return st;
#endif
  } else if (p.light_ok) {
    if ((st = allow_max_dyn_smem (light_kernel_for (p))) != B200_OK) return st;
  } else if (p.ntap_ok) {
    if ((st = prepare_ntap (p, &h->ntap)) != B200_OK) return st;
  }
  return B200_OK;
}

int ensure_pipeline (b200_vcs * h, int chunk)
{
  if (h->pipeline_ready && chunk <= h->slot_frames) return B200_OK;
  h->in_bytes = b200_video_info_size (&h->plan.in);
  h->out_bytes = b200_video_info_size (&h->plan.frame_out);
  if (!h->pipeline_ready) {
    B200_CUDA_TRY (cudaStreamCreateWithFlags (&h->s_h2d, cudaStreamNonBlocking));
    B200_CUDA_TRY (cudaStreamCreateWithFlags (&h->s_run, cudaStreamNonBlocking));
    B200_CUDA_TRY (cudaStreamCreateWithFlags (&h->s_d2h, cudaStreamNonBlocking));
    for (int i = 0; i < b200_vcs::kSlots; i++) {
      B200_CUDA_TRY (cudaEventCreateWithFlags (&h->ev_in[i], cudaEventDisableTiming));
      B200_CUDA_TRY (cudaEventCreateWithFlags (&h->ev_run[i], cudaEventDisableTiming));
      B200_CUDA_TRY (cudaEventCreateWithFlags (&h->ev_out[i], cudaEventDisableTiming));
    }
    h->pipeline_ready = true;
  }
  // (re)size the slots: each holds `chunk` frames, so that one kernel launch and one event triple serve a whole chunk
  for (int i = 0; i < b200_vcs::kSlots; i++) {
    B200_CUDA_TRY (cudaFree (h->slot_in[i])); h->slot_in[i] = nullptr;       // cudaFree waits for work still using it
    B200_CUDA_TRY (cudaFree (h->slot_out[i])); h->slot_out[i] = nullptr;
  }
  h->slot_frames = 0;
  for (int i = 0; i < b200_vcs::kSlots; i++) {
    B200_CUDA_TRY (cudaMalloc ((void **) &h->slot_in[i], h->in_bytes * chunk));
    B200_CUDA_TRY (cudaMalloc ((void **) &h->slot_out[i], h->out_bytes * chunk));
  }
  h->slot_frames = chunk;
  return B200_OK;
}

}  // namespace

namespace b200 {

bool vcs_comp_fusable (const b200_vcs * h)
{
  const VcsPlan & p = h->plan;
  const VideoFormatDesc & d = *video_format (p.out.format);
  return h->device >= 0 && p.planes_mode && !p.has_dest && (d.family == FAMILY_YUV420 || d.family == FAMILY_NV) && d.bytes == 1;
}

int vcs_device (const b200_vcs * h) { return h->device; }
const b200_video_info & vcs_in_info (const b200_vcs * h) { return h->plan.in; }
const b200_video_info & vcs_out_info (const b200_vcs * h) { return h->plan.frame_out; }

int vcs_comp_launch (b200_vcs * h, int n, const uint8_t *const *in, uint8_t * dst, const b200_video_info & di,
    const CompStore & S, cudaStream_t stream)
{
  if (!vcs_comp_fusable (h) || n < 1 || n > B200_VCS_MAX_BATCH) return B200_ERR_STATE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  VcsBatch b;
  for (int i = 0; i < n; i++) { b.in[i] = in[i]; b.out[i] = dst; }
  unsigned long long off[3];
  int stride[3];
  for (int k = 0; k < 3; k++) { off[k] = di.offset[k]; stride[k] = di.stride[k]; }
  return launch_planes_comp (h->planes, b, n, stream, alignment (b.in, n) >= 8, off, stride, S);
}

}  // namespace b200

extern "C" {

void b200_vcs_config_init (b200_vcs_config * cfg)
{
  if (!cfg) return;
  memset (cfg, 0, sizeof (*cfg));
  cfg->method = B200_SCALE_BILINEAR;    // DEFAULT_PROP_METHOD, gstvideoconvertscale.c:130
  cfg->envelope = 2.0; cfg->sharpness = 1.0; cfg->sharpen = 0.0;
  cfg->border_argb = 0xff000000u; cfg->fill_border = 1;   // DEFAULT_OPT_FILL_BORDER / _BORDER_ARGB, video-converter.c:778, :782
}

// video-info.c:882-894 (packed), :997-1063 (8-bit planar and semi-planar), :1142-1188 (10 / 12 / 16 bits); RGBP / BGRP
// are laid out like Y444 (:1030-1041)
int b200_video_info_set_format (b200_video_info * info, int format, int width, int height)
{
  if (!info || width < 1 || height < 1) return B200_ERR_INVALID_ARG;
  memset (info, 0, sizeof (*info));
  info->format = format; info->width = width; info->height = height;
  const VideoFormatDesc *d = video_format (format);
  if (!d) return B200_ERR_UNSUPPORTED;
  if (d->n_planes == 1) {
    info->stride[0] = (width * (d->family == FAMILY_RGB ? 4 : 2) + 3) & ~3;
  } else {
    const int cw = (width + (1 << d->wsub) - 1) >> d->wsub, rows = luma_rows (*d, height);
    info->stride[0] = (width * d->bytes + 3) & ~3;
    info->stride[1] = d->family == FAMILY_NV ? info->stride[0] : (cw * d->bytes + 3) & ~3;
    info->offset[1] = (uint64_t) info->stride[0] * rows;
    if (d->n_planes == 3) {
      info->stride[2] = info->stride[1];
      info->offset[2] = info->offset[1] + (uint64_t) info->stride[1] * (rows >> d->hsub);
    }
  }
  fill_colorimetry (info, *d, height);
  return B200_OK;
}

size_t b200_video_info_size (const b200_video_info * info)
{
  if (!info) return 0;
  const VideoFormatDesc *d = video_format (info->format);
  if (!d || d->n_planes == 1) return (size_t) info->offset[0] + (size_t) info->stride[0] * info->height;
  const int rows = luma_rows (*d, info->height);
  auto end = [&] (int k) { return (size_t) info->offset[k] + (size_t) info->stride[k] * (k ? rows >> d->hsub : rows); };
  if (d->family == FAMILY_RGBP) return std::max ({end (0), end (1), end (2)});      // three full planes in any order
  if (d->family == FAMILY_YUV420 && d->bytes == 1) return std::max (end (1), end (2));   // either chroma plane last
  return end (d->n_planes - 1);
}

int b200_vcs_create (const b200_video_info * in, const b200_video_info * out,
    const b200_vcs_config * cfg, int device, b200_vcs ** handle)
{
  if (!handle) return B200_ERR_INVALID_ARG;
  *handle = nullptr;
  b200_vcs_config defcfg;
  if (!cfg) { b200_vcs_config_init (&defcfg); cfg = &defcfg; }
  b200_vcs *h = new (std::nothrow) b200_vcs ();
  if (!h) return B200_ERR_NOMEM;
  int st = build_vcs_plan (in, out, cfg, &h->plan);
  if (st != B200_OK) { delete h; return st; }
  if (h->plan.has_dest) {
    // per-plane rectangles: chroma planes use GST_VIDEO_FORMAT_INFO_SCALE_WIDTH / _HEIGHT (round up), :7209-7221
    const VcsPlan & q = h->plan;
    const b200_video_info & f = q.frame_out;
    BorderDev & b = h->border;
    memset (&b, 0, sizeof (b));
    const VideoFormatDesc & d = *video_format (f.format);
    if (q.rgbp_out) {                                               // pack_RGBP of the border line: each plane its own byte
      b.n_planes = 3;
      for (int k = 0; k < 3; k++)
        b.pl[k] = BorderPlane {f.offset[k], f.stride[k], f.width, f.height, 1, q.dest[0], q.dest[1], q.dest[2], q.dest[3], (unsigned) q.border_px[k]};
    } else if (d.family == FAMILY_RGB) {
      b.n_planes = 1;
      b.pl[0] = BorderPlane {f.offset[0], f.stride[0], f.width, f.height, 4, q.dest[0], q.dest[1], q.dest[2], q.dest[3],
        (unsigned) q.border_px[0] | ((unsigned) q.border_px[1] << 8) | ((unsigned) q.border_px[2] << 16) | ((unsigned) q.border_px[3] << 24)};
    } else {
      const int cx = (q.dest[0] + 1) / 2, cy = (q.dest[1] + 1) / 2, cw = (q.dest[2] + 1) / 2, chh = (q.dest[3] + 1) / 2;
      const int CW = (f.width + 1) / 2, CH = (f.height + 1) / 2;
      b.pl[0] = BorderPlane {f.offset[0], f.stride[0], f.width, f.height, 1, q.dest[0], q.dest[1], q.dest[2], q.dest[3], (unsigned) q.border_yuv[0]};
      const int pu = d.plane_u, pv = d.plane_v;
      b.n_planes = d.n_planes;
      if (d.family == FAMILY_YUV420) {
        b.pl[1] = BorderPlane {f.offset[pu], f.stride[pu], CW, CH, 1, cx, cy, cw, chh, (unsigned) q.border_yuv[1]};
        b.pl[2] = BorderPlane {f.offset[pv], f.stride[pv], CW, CH, 1, cx, cy, cw, chh, (unsigned) q.border_yuv[2]};
      } else {                                                      // one interleaved pair: U at byte u_index
        const unsigned u = (unsigned) q.border_yuv[1], v = (unsigned) q.border_yuv[2];
        b.pl[1] = BorderPlane {f.offset[pu], f.stride[pu], CW, CH, 2, cx, cy, cw, chh, u << (8 * d.u_index) | v << (8 - 8 * d.u_index)};
      }
    }
  }
  h->knobs = read_knobs ();
  VcsPlan & p = h->plan;
  if (!p.planes_mode && !p.in_422_444 && (!p.yuv_out || (!p.rgb_in && !p.has_dest))) {
    // the exact-2:1 kernel: the one kernel of a packed or planar RGB output, or the first launch of the 4:2:0 chain
    h->l2_tables = build_lanczos2_tables (p);
    h->l2v2_tables = build_lanczos2_v2_tables (p, h->l2_tables);
    // planar (I420 / YV12) input, planar RGB output and the chain (matrix stage off) exist in the second form only;
    // the first form and the tensor forms (variants 6 / 7) decline planar RGB output
    const bool v2 = h->l2v2_tables.ok && !h->knobs.l2_v1 && !h->knobs.l2_x4;
    const bool v2_only = p.planar || p.rgbp_out;
    p.lanczos2_ok = h->l2_tables.ok && (p.yuv_out ? v2 && !h->knobs.cross_generic : (!v2_only || v2));
    if (!p.yuv_out && !p.rgbp_out) {
      h->mma_tables = build_l2mma_tables (p);
#ifndef B200_CUDA_EMU
      h->tc_tables = build_l2tc_tables (p, h->l2_tables);
#endif
    }
  }
  if (!p.planes_mode && !p.yuv_out && !p.rgbp_out && ((p.out.stride[0] & 3) || (p.out.offset[0] & 3))) { delete h; return B200_ERR_UNSUPPORTED; }
  h->device = device;
  h->deint_scaled = p.planes_mode && p.rgbp_out && p.planes[0].mode == PM_SCALE;
  if (device >= 0) {
    int ndev = b200_device_count ();
    if (ndev <= 0) { delete h; return ndev < 0 ? ndev : B200_ERR_NO_DEVICE; }
    if (device >= ndev) { delete h; return B200_ERR_INVALID_ARG; }
    DeviceGuard g (device);
    if (!g.ok) { delete h; return B200_ERR_CUDA; }
    if ((st = prepare_device (h)) != B200_OK) { b200_vcs_destroy (h); return st; }
  }
  // the kernel this plan will run (also reported for host-only handles: caps negotiation dry-runs, CPU tests).  Variant 6
  // (mma.sync formulation of the 2:1 kernel) is not timed on the H100 and not the default: kept selectable through
  // b200_vcs_set_kernel_variant for cross-checks only
  h->variant = default_variant (h);
  *handle = h;
  return B200_OK;
}

void b200_vcs_destroy (b200_vcs * h)
{
  if (!h) return;
  if (h->device >= 0) {
    DeviceGuard g (h->device);
    cudaFree (h->d_hoff); cudaFree (h->d_voff); cudaFree (h->d_hcoef); cudaFree (h->d_vcoef);
    cudaFree (h->d_hsum); cudaFree (h->d_vsum); cudaFree (h->d_cmode);
    cudaFree (h->l2.d_htab); cudaFree (h->l2.d_vtab); cudaFree (h->ntap.d_h); cudaFree (h->ntap.d_v);
    cudaFree (h->l2.d_htab4); cudaFree (h->l2.d_vtab4); cudaFree (h->l2.d_v4); cudaFree (h->l2v2.d_vkind);
    cudaFree (h->mma.d_bh); cudaFree (h->mma.d_bv); cudaFree (h->mma.d_h4); cudaFree (h->mma.d_v4);
#ifndef B200_CUDA_EMU
    cudaFree (h->tc.d_band); cudaFree (h->tc.d_vband); cudaFree (h->tc.d_hx4); cudaFree (h->tc.d_vx4);
#endif
    free_planes (&h->planes);
    free_plane_fast (&h->rgb420_scaler);
    cudaFree (h->d_scratch);
    for (int i = 0; i < b200_vcs::kSlots; i++) {
      cudaFree (h->slot_in[i]); cudaFree (h->slot_out[i]);
      if (h->ev_in[i]) cudaEventDestroy (h->ev_in[i]);
      if (h->ev_run[i]) cudaEventDestroy (h->ev_run[i]);
      if (h->ev_out[i]) cudaEventDestroy (h->ev_out[i]);
    }
    if (h->s_h2d) cudaStreamDestroy (h->s_h2d);
    if (h->s_run) cudaStreamDestroy (h->s_run);
    if (h->s_d2h) cudaStreamDestroy (h->s_d2h);
  }
  delete h;
}

int b200_vcs_convert_batch (b200_vcs * h, int n, const void *const *in_frames,
    void *const *out_frames, void *cuda_stream)
{
  if (!h || !in_frames || !out_frames || n < 1 || n > B200_VCS_MAX_BATCH) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  VcsBatch b;
  for (int i = 0; i < n; i++) {
    if (!in_frames[i] || !out_frames[i]) return B200_ERR_INVALID_ARG;
    b.in[i] = (const uint8_t *) in_frames[i];
    b.out[i] = (uint8_t *) out_frames[i];
  }
  return launch_convert (h, n, b, (cudaStream_t) cuda_stream);
}

int b200_vcs_convert (b200_vcs * h, const void *in_frame, void *out_frame, void *cuda_stream)
{
  return b200_vcs_convert_batch (h, 1, &in_frame, &out_frame, cuda_stream);
}

int b200_vcs_convert_host (b200_vcs * h, int n, const void *const *in_host, void *const *out_host)
{
  if (!h || !in_host || !out_host || n < 1) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  for (int i = 0; i < n; i++) if (!in_host[i] || !out_host[i]) return B200_ERR_INVALID_ARG;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  // Three-stage software pipeline over kSlots device slots of `chunk` frames: the upload of chunk c+1 and the download
  // of chunk c-1 overlap the kernel of chunk c (the copy engines run beside the SMs).  One kernel launch and one event
  // triple per chunk, not per frame; with few frames the chunk shrinks so that all three stages still overlap.
  const int K = b200_vcs::kSlots;
  // chunks only for long calls: with few frames per call the pipeline's fill and drain would outweigh what chunking saves
  const int chunk = n >= 16 * b200_vcs::kChunk ? b200_vcs::kChunk : (n >= 32 ? 2 : 1);
  int st = ensure_pipeline (h, chunk);
  if (st != B200_OK) return st;
  int c = 0;
  for (int i0 = 0; i0 < n; i0 += chunk, c++) {
    const int s = c % K, m = min (chunk, n - i0);
    if (c >= K) {
      B200_CUDA_TRY (cudaStreamWaitEvent (h->s_h2d, h->ev_run[s], 0));   // input slot consumed
      B200_CUDA_TRY (cudaStreamWaitEvent (h->s_run, h->ev_out[s], 0));   // output slot drained
    }
    VcsBatch b;
    for (int j = 0; j < m; j++) {
      b.in[j] = h->slot_in[s] + (size_t) j * h->in_bytes; b.out[j] = h->slot_out[s] + (size_t) j * h->out_bytes;
      B200_CUDA_TRY (cudaMemcpyAsync ((void *) b.in[j], in_host[i0 + j], h->in_bytes, cudaMemcpyHostToDevice, h->s_h2d));
    }
    B200_CUDA_TRY (cudaEventRecord (h->ev_in[s], h->s_h2d));
    B200_CUDA_TRY (cudaStreamWaitEvent (h->s_run, h->ev_in[s], 0));
    if ((st = launch_convert (h, m, b, h->s_run)) != B200_OK) return st;
    B200_CUDA_TRY (cudaEventRecord (h->ev_run[s], h->s_run));
    B200_CUDA_TRY (cudaStreamWaitEvent (h->s_d2h, h->ev_run[s], 0));
    for (int j = 0; j < m; j++)
      B200_CUDA_TRY (cudaMemcpyAsync (out_host[i0 + j], b.out[j], h->out_bytes, cudaMemcpyDeviceToHost, h->s_d2h));
    B200_CUDA_TRY (cudaEventRecord (h->ev_out[s], h->s_d2h));
  }
  B200_CUDA_TRY (cudaStreamSynchronize (h->s_d2h));
  return B200_OK;
}

int b200_vcs_copy_probe (b200_vcs * h, int n, const void *const *in_host, void *const *out_host)
{
  // the copies of b200_vcs_convert_host without the kernels: H2D of every input on one stream, D2H of every output
  // (whatever the slots hold) on another, both directions in flight together - the link's ceiling for this call
  if (!h || !in_host || !out_host || n < 1) return B200_ERR_INVALID_ARG;
  if (h->device < 0) return B200_ERR_NO_DEVICE;
  DeviceGuard g (h->device);
  if (!g.ok) return B200_ERR_CUDA;
  int st = ensure_pipeline (h, max (h->slot_frames, 1));
  if (st != B200_OK) return st;
  const int K = b200_vcs::kSlots, chunk = h->slot_frames;
  for (int i = 0; i < n; i++) {
    const int s = (i / chunk) % K, j = i % chunk;
    if (!in_host[i] || !out_host[i]) return B200_ERR_INVALID_ARG;
    B200_CUDA_TRY (cudaMemcpyAsync (h->slot_in[s] + (size_t) j * h->in_bytes, in_host[i], h->in_bytes, cudaMemcpyHostToDevice, h->s_h2d));
    B200_CUDA_TRY (cudaMemcpyAsync (out_host[i], h->slot_out[s] + (size_t) j * h->out_bytes, h->out_bytes, cudaMemcpyDeviceToHost, h->s_d2h));
  }
  B200_CUDA_TRY (cudaStreamSynchronize (h->s_h2d));
  B200_CUDA_TRY (cudaStreamSynchronize (h->s_d2h));
  return B200_OK;
}

int b200_vcs_get_plan_info (const b200_vcs * h, b200_vcs_plan_info * info)
{
  if (!h || !info) return B200_ERR_INVALID_ARG;
  const VcsPlan & p = h->plan;
  memset (info, 0, sizeof (*info));
  info->h_taps = p.h.scaling ? p.h.n_taps : 0;
  info->v_taps = p.v.scaling ? p.v.n_taps : 0;
  info->h_first = p.h_first; info->matrix_first = p.matrix_first;
  for (int i = 0; i < 5; i++) info->p[i] = p.p[i];
  info->tile_w = p.tile_w; info->tile_h = p.tile_h; info->smem_bytes = p.smem_bytes;
  const Route r = select_route (h, h->variant, 16, 16);
  info->kernel_variant = r.kernel_variant;
  info->n_launches_per_convert = r.n_launches;
  return B200_OK;
}

int b200_vcs_get_taps (const b200_vcs * h, int dir, uint32_t * offsets, int16_t * taps,
    size_t offsets_len, size_t taps_len)
{
  if (!h || (dir != 0 && dir != 1)) return B200_ERR_INVALID_ARG;
  const AxisPlan & a = dir == 0 ? h->plan.h : h->plan.v;
  if (offsets) {
    if (offsets_len < a.offset.size ()) return B200_ERR_INVALID_ARG;
    memcpy (offsets, a.offset.data (), a.offset.size () * sizeof (uint32_t));
  }
  if (taps) {
    if (taps_len < a.coef.size ()) return B200_ERR_INVALID_ARG;
    memcpy (taps, a.coef.data (), a.coef.size () * sizeof (int16_t));
  }
  return (int) a.coef_per_out;
}

int b200_vcs_get_matrix (const b200_vcs * h, int32_t im[16])
{
  if (!h || !im) return B200_ERR_INVALID_ARG;
  const VcsPlan & p = h->plan;
  const bool has = !p.planes_mode && (!p.yuv_out || p.rgb_in);
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) im[4 * i + j] = has ? p.im[i][j] : 0;
  return B200_OK;
}

int b200_vcs_get_chroma_plan (const b200_vcs * h, uint8_t * mode, size_t len)
{
  if (!h || !mode || len < h->plan.chroma_mode.size ()) return B200_ERR_INVALID_ARG;
  memcpy (mode, h->plan.chroma_mode.data (), h->plan.chroma_mode.size ());
  return B200_OK;
}

int b200_vcs_set_kernel_variant (b200_vcs * h, int variant)
{
  if (!h || variant < 0 || (variant > 3 && variant != 6 && variant != 7)) return B200_ERR_INVALID_ARG;
  // eligible: a one-kernel route that takes the variant's kernel on aligned frames.  A host-only handle has no n-tap
  // tables to run variant 3 with.
  const Route r = select_route (h, variant, 16, 16);
  if (r.path != Path::one || r.named_variant != variant || (variant == 3 && h->device < 0)) return B200_ERR_UNSUPPORTED;
  h->variant = variant;
  return B200_OK;
}

const char *b200_vcs_kernel_name (const b200_vcs * h)
{
  return h ? select_route (h, h->variant, 16, 16).name : "";
}

}  // extern "C"
