"""ctypes bindings of the CPU checkers — TEST INFRASTRUCTURE ONLY.

  liboracle.so        oracle/*.c, our plain-C restatement of the reference algorithm
  _ref/libgstref.so   the reference's own sources compiled in place (oracle/Makefile);
                      prebuilt here, travels to the GPU box, never rebuilt there

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs import this module.
Nothing under gstreamer_b200/ does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "liboracle.so")
REF_SO = os.path.join(_HERE, "_ref", "libgstref.so")

# element method -> (GstVideoResamplerMethod, max-taps option, (cubic b, c))
# gst/videoconvertscale/gstvideoconvertscale.c:991-1050
ELEMENT_METHODS = {0: (0, 0, None), 1: (1, 2, None), 2: (3, 4, None), 3: (4, 0, None), 4: (1, 0, None),
                   5: (3, 0, None), 6: (2, 0, (0., 0.)), 7: (2, 0, (1., 0.)), 8: (2, 0, (0., .5)),
                   9: (2, 0, (1 / 3, 1 / 3))}
FMT = {"RGBx": 7, "BGRx": 8, "xRGB": 9, "xBGR": 10, "RGBA": 11, "BGRA": 12, "ARGB": 13, "ABGR": 14,
       "AYUV": 6, "NV12": 23, "NV21": 24, "I420": 2, "YV12": 3, "YUY2": 4, "UYVY": 5, "Y42B": 18, "YVYU": 19, "Y444": 20}


def build(ref=True):
    """(re)build the checkers with oracle/Makefile; its ref and refcuda targets build only where REFROOT holds the
    reference's sources and say so otherwise"""
    subprocess.check_call(["make", "-s", "-C", _HERE, "oracle"])
    if ref:
        subprocess.check_call(["make", "-s", "-C", _HERE, "ref"])
        # the reference's CUDA converter kernel as bench.py's gpu_baseline (needs nvcc; a missing compiler is not fatal)
        subprocess.call(["make", "-s", "-C", _HERE, "refcuda"])


REFCUDA_BENCH = os.path.join(_HERE, "_ref", "refcuda_bench")


def run_refcuda_bench(reps=20, timeout=120):
    """runs the reference's own CUDA converter kernel (oracle/_ref/refcuda_bench) on the bench shape; None if absent"""
    import json
    if not os.path.exists(REFCUDA_BENCH):
        return None
    try:
        out = subprocess.run([REFCUDA_BENCH, str(reps)], capture_output=True, text=True, timeout=timeout)
        return json.loads(out.stdout.strip().splitlines()[-1])
    except Exception as e:
        return {"error": repr(e)}


class RS(C.Structure):
    _fields_ = [("method", C.c_int), ("max_taps_opt", C.c_int), ("n_taps_req", C.c_int),
                ("envelope", C.c_double), ("sharpness", C.c_double), ("sharpen", C.c_double),
                ("cubic_b", C.c_double), ("cubic_c", C.c_double)]


class VcsDesc(C.Structure):
    _fields_ = [("in_format", C.c_int), ("in_width", C.c_int), ("in_height", C.c_int),
                ("in_stride", C.c_int * 4), ("in_offset", C.c_size_t * 4), ("in_matrix", C.c_int),
                ("in_range", C.c_int), ("in_chroma_site", C.c_int), ("out_format", C.c_int),
                ("out_width", C.c_int), ("out_height", C.c_int), ("out_stride", C.c_int * 4),
                ("out_offset", C.c_size_t * 4), ("rs", RS),
                ("out_matrix", C.c_int), ("out_chroma_site", C.c_int), ("out_range", C.c_int), ("force_resample", C.c_int)]


class OraclePad(C.Structure):
    _fields_ = [("data", C.c_void_p), ("width", C.c_int), ("height", C.c_int), ("stride", C.c_int),
                ("xpos", C.c_int), ("ypos", C.c_int), ("alpha", C.c_double), ("op", C.c_int)]


_oracle = None
_ref = None


def oracle():
    global _oracle
    if _oracle is None:
        if not os.path.exists(ORACLE_SO):
            build(ref=False)
        o = C.CDLL(ORACLE_SO)
        P = C.c_void_p
        o.oracle_resampler_taps.argtypes = [C.POINTER(RS), C.c_int, C.c_int, P, P]
        o.oracle_quantize_taps.argtypes = [P, P, C.c_int, C.c_int]
        o.oracle_vcs_default_desc.argtypes = [C.POINTER(VcsDesc)] + [C.c_int] * 8
        o.oracle_vcs_in_size.restype = C.c_size_t
        o.oracle_vcs_in_size.argtypes = [C.POINTER(VcsDesc)]
        o.oracle_vcs_out_size.restype = C.c_size_t
        o.oracle_vcs_out_size.argtypes = [C.POINTER(VcsDesc)]
        o.oracle_vcs_matrix.argtypes = [C.POINTER(VcsDesc), P, P]
        o.oracle_vcs_convert.argtypes = [C.POINTER(VcsDesc), P, P]
        o.oracle_vcs_matrix_rgb2yuv.argtypes = [C.POINTER(VcsDesc), P]
        o.oracle_vcs_borders.argtypes = [C.c_int] * 4 + [P]
        o.oracle_vcs_borders.restype = None
        o.oracle_vcs_convert_dest.argtypes = [C.POINTER(VcsDesc)] + [C.c_int] * 4 + [C.c_uint32, P, P]
        if hasattr(o, "oracle_compositor"):
            o.oracle_compositor.argtypes = [C.c_int, P, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.POINTER(OraclePad), C.c_int]
        if hasattr(o, "oracle_compositor_yuv"):
            o.oracle_compositor_yuv_size.restype = C.c_size_t
            o.oracle_compositor_yuv_size.argtypes = [C.c_int] * 3
            o.oracle_compositor_yuv.argtypes = [C.c_int, P, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(OraclePad), C.c_int]
        if hasattr(o, "oracle_ars_new"):
            o.oracle_ars_new.restype = P
            o.oracle_ars_new.argtypes = [C.c_int] * 4
            o.oracle_ars_new_fmt.restype = P
            o.oracle_ars_new_fmt.argtypes = [C.c_int] * 5
            o.oracle_ars_new_opts.restype = P
            o.oracle_ars_new_opts.argtypes = [C.c_int] * 8
            o.oracle_ars_process_any.restype = C.c_size_t
            o.oracle_ars_process_any.argtypes = [P, P, C.c_size_t, P, C.c_size_t]
            o.oracle_ars_free.argtypes = [P]
            o.oracle_ars_reset.argtypes = [P]
            if hasattr(o, "oracle_ars_update"):
                o.oracle_ars_update.argtypes = [P, C.c_int, C.c_int]
            for n in ("oracle_ars_get_out_frames", "oracle_ars_get_in_frames"):
                getattr(o, n).restype = C.c_size_t
                getattr(o, n).argtypes = [P, C.c_size_t]
            o.oracle_ars_max_latency.restype = C.c_size_t
            o.oracle_ars_max_latency.argtypes = [P]
            o.oracle_ars_process.restype = C.c_size_t
            o.oracle_ars_process.argtypes = [P, P, C.c_size_t, P, C.c_size_t]
            o.oracle_ars_info.argtypes = [P] + [C.POINTER(C.c_int)] * 6
            o.oracle_ars_phase_taps.argtypes = [P, C.c_int, P]
        _oracle = o
    return _oracle


def have_ref():
    return os.path.exists(REF_SO)


def ref():
    global _ref
    if _ref is None:
        r = C.CDLL(REF_SO)
        P = C.c_void_p
        r.ref_vcs_new.restype = P
        if hasattr(r, 'ref_vcs_next_dest'):
            r.ref_vcs_next_dest.argtypes = [C.c_int] * 4
            r.ref_vcs_next_dest.restype = None
            r.ref_vcs_next_border_argb.argtypes = [C.c_uint]
            r.ref_vcs_next_border_argb.restype = None
        r.ref_vcs_new.argtypes = ([C.c_int] * 3 + [P] * 2 + [C.c_int] * 3) * 2 + [C.c_int] * 3 + [C.c_double] * 3
        r.ref_vcs_convert.argtypes = [P, P, P]
        r.ref_vcs_free.argtypes = [P]
        r.ref_scaler_taps.argtypes = [C.c_int] * 4 + [C.c_double] * 3 + [P, P, P]
        if hasattr(r, "ref_compositor"):
            r.ref_compositor.argtypes = [C.c_int, P, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.POINTER(OraclePad), C.c_int]
        if hasattr(r, "ref_compositor_yuv"):
            r.ref_compositor_yuv.argtypes = [C.c_int, P, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(OraclePad), C.c_int]
        if hasattr(r, "ref_ars_new"):
            r.ref_ars_new.restype = P
            r.ref_ars_new.argtypes = [C.c_int] * 4
            if hasattr(r, "ref_ars_new_fmt"):
                r.ref_ars_new_fmt.restype = P
                r.ref_ars_new_fmt.argtypes = [C.c_int] * 5
            if hasattr(r, "ref_ars_new_opts"):
                r.ref_ars_new_opts.restype = P
                r.ref_ars_new_opts.argtypes = [C.c_int] * 8
            r.ref_ars_free.argtypes = [P]
            r.ref_ars_reset.argtypes = [P]
            if hasattr(r, "ref_ars_update"):
                r.ref_ars_update.argtypes = [P] + [C.c_int] * 6
            for n in ("ref_ars_get_out_frames", "ref_ars_get_in_frames"):
                getattr(r, n).restype = C.c_size_t
                getattr(r, n).argtypes = [P, C.c_size_t]
            r.ref_ars_max_latency.restype = C.c_size_t
            r.ref_ars_max_latency.argtypes = [P]
            r.ref_ars_process.restype = C.c_size_t
            r.ref_ars_process.argtypes = [P, P, C.c_size_t, P, C.c_size_t]
            r.ref_ars_info.argtypes = [P] + [C.POINTER(C.c_int)] * 6
            r.ref_ars_phase_taps.argtypes = [P, C.c_int, P]
        _ref = r
    return _ref


# ----------------------------------------------------------------------------- video
def vcs_desc(iw, ih, ow, oh, method, in_fmt=23, out_fmt=12, site=None, matrix=None, rng=None):
    d = VcsDesc()
    m, mt, bc = ELEMENT_METHODS[int(method)]
    st = oracle().oracle_vcs_default_desc(C.byref(d), in_fmt, iw, ih, out_fmt, ow, oh, m, mt)
    if st != 0:
        raise ValueError("oracle_vcs_default_desc failed")
    if bc:
        d.rs.cubic_b, d.rs.cubic_c = bc
    if site is not None:
        d.in_chroma_site = int(site)
    if matrix is not None:
        d.in_matrix = int(matrix)
    if rng is not None:
        d.in_range = int(rng)
    return d


def vcs_sizes(d):
    return oracle().oracle_vcs_in_size(C.byref(d)), oracle().oracle_vcs_out_size(C.byref(d))


def oracle_vcs_convert(d, frame):
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    isz, osz = vcs_sizes(d)
    assert frame.size >= isz
    out = np.zeros(osz, dtype=np.uint8)
    st = oracle().oracle_vcs_convert(C.byref(d), frame.ctypes.data, out.ctypes.data)
    if st != 0:
        raise RuntimeError(f"oracle_vcs_convert -> {st}")
    return out


class RefVcs:
    """The reference's own GstVideoConverter (compiled in place), element option mapping."""

    def __init__(self, iw, ih, ow, oh, method, in_fmt=23, out_fmt=12, site=-1, matrix=-1, rng=-1,
                 n_threads=1, out_matrix=-1, out_rng=-1, out_site=-1, dest=None, border_argb=None):
        if border_argb is not None:
            ref().ref_vcs_next_border_argb(int(border_argb))
        if dest is not None:
            ref().ref_vcs_next_dest(*[int(v) for v in dest])
        self.h = ref().ref_vcs_new(in_fmt, iw, ih, None, None, matrix, rng, site,
                                   out_fmt, ow, oh, None, None, out_matrix, out_rng, out_site,
                                   int(method), n_threads, 4, 2.0, 1.0, 0.0)
        if not self.h:
            raise RuntimeError("ref_vcs_new failed")
        self.out_bytes = ow * oh * 4

    def convert(self, frame, out=None):
        frame = np.ascontiguousarray(frame, dtype=np.uint8)
        if out is None:
            out = np.zeros(self.out_bytes, dtype=np.uint8)
        ref().ref_vcs_convert(self.h, frame.ctypes.data, out.ctypes.data)
        return out

    def close(self):
        if self.h:
            ref().ref_vcs_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def vcs_borders(iw, ih, ow, oh):
    """the element's add-borders rectangle (x, y, w, h) for pixel aspect ratio 1/1 on both sides"""
    d = (C.c_int * 4)()
    oracle().oracle_vcs_borders(iw, ih, ow, oh, d)
    return tuple(d)


def oracle_vcs_convert_dest(d, frame, dest, border_argb=0xff000000, fill=0):
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    out = np.full(vcs_sizes(d)[1], fill, dtype=np.uint8)
    st = oracle().oracle_vcs_convert_dest(C.byref(d), dest[0], dest[1], dest[2], dest[3], border_argb, frame.ctypes.data,
                                          out.ctypes.data)
    if st != 0:
        raise RuntimeError(f"oracle_vcs_convert_dest -> {st}")
    return out


# ------------------------------------------------------------------- synthetic inputs
def lcg_bytes(n, seed):
    """videotestsrc's noise generator (gst/videotestsrc/videotestsrc.c random_char):
    s = s*1103515245 + 12345; (s >> 16) & 0xff — vectorised by jumping the LCG."""
    a, c, m = 1103515245, 12345, 1 << 32
    # state_k = a^k * s0 + c*(a^k - 1)/(a - 1)  (mod 2^32): build by doubling
    out = np.empty(n, dtype=np.uint32)
    state = np.uint64(seed & 0xffffffff)
    # generate in chunks with a scalar loop over a small block then affine jumps
    block = 1 << 12
    first = np.empty(min(block, n), dtype=np.uint64)
    s = int(seed) & 0xffffffff
    for i in range(first.size):
        s = (s * a + c) % m
        first[i] = s
    out[:first.size] = first
    if n > block:
        # affine map for a jump of `block` steps
        A, Cc = 1, 0
        for _ in range(block):
            A, Cc = (A * a) % m, (Cc * a + c) % m
        cur = first.copy()
        pos = block
        while pos < n:
            cur = (cur * np.uint64(A) + np.uint64(Cc)) % np.uint64(m)
            k = min(block, n - pos)
            out[pos:pos + k] = cur[:k]
            pos += k
    del state
    return ((out >> 16) & 0xff).astype(np.uint8)


def nv12_random_frame(w, h, seed):
    """uniform random Y,U,V bytes in the default NV12 layout (SURVEY §8d generator ii)"""
    stride = (w + 3) & ~3
    rows = ((h + 1) & ~1) + ((h + 1) & ~1) // 2
    return lcg_bytes(stride * rows, seed + 1)


# audio sample formats: (oracle enum, GstAudioFormat value, numpy dtype, amplitude for test signals)
AUDIO_FORMATS = {"F32": (0, 28, np.float32, 0.5), "S16": (1, 4, np.int16, 9000.0), "S32": (2, 12, np.int32, 6e8),
                 "F64": (3, 30, np.float64, 0.5)}


def audio_test_signal(rng, n, ch, fmt):
    _, _, dt, amp = AUDIO_FORMATS[fmt]
    x = rng.standard_normal((n, ch)) * amp
    if np.issubdtype(dt, np.integer):
        x = np.clip(x, np.iinfo(dt).min, np.iinfo(dt).max)
    return x.astype(dt)


def i420_random_frame(w, h, seed):
    """uniform random Y,U,V bytes in the default I420 / YV12 layout (video-info.c:997-1009)"""
    sy = (w + 3) & ~3
    sc = ((((w + 1) & ~1) // 2) + 3) & ~3
    hh = (h + 1) & ~1
    return lcg_bytes(sy * hh + 2 * sc * (hh // 2), seed + 1)


def nv12_smpte_like_frame(w, h, seed=0):
    """structured frame in the spirit of videotestsrc's smpte pattern: 7 vertical bars over the
    top 2/3, a reverse strip, then a ramp / noise quarter (gst/videotestsrc/videotestsrc.c:382-481)"""
    stride = (w + 3) & ~3
    hh = (h + 1) & ~1
    y = np.zeros((hh, stride), dtype=np.uint8)
    uv = np.zeros((hh // 2, stride), dtype=np.uint8)
    bars_y = [180, 162, 131, 112, 84, 65, 35]
    bars_u = [128, 44, 156, 72, 184, 100, 212]
    bars_v = [128, 142, 44, 58, 198, 212, 114]
    xs = (np.arange(stride) * 7 // max(w, 1)).clip(0, 6)
    y[:] = np.array(bars_y, dtype=np.uint8)[xs]
    cx = (np.arange(stride // 2) * 2 * 7 // max(w, 1)).clip(0, 6)
    uv[:, 0::2] = np.array(bars_u, dtype=np.uint8)[cx][: uv[:, 0::2].shape[1]]
    uv[:, 1::2] = np.array(bars_v, dtype=np.uint8)[cx][: uv[:, 1::2].shape[1]]
    y0 = 2 * h // 3
    y1 = 3 * h // 4
    y[y0:y1] = y[y0:y1, ::-1]
    y[y1:] = (np.arange(stride) * 255 // max(w - 1, 1)).astype(np.uint8)
    noise = lcg_bytes(stride * (hh - y1), seed).reshape(hh - y1, stride)
    y[y1:, w // 2:] = noise[:, w // 2:]
    uv[y1 // 2:] = 128
    return np.concatenate([y.reshape(-1), uv.reshape(-1)])
