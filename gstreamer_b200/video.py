"""Host-side mirror of the reference's convert+scale interface over the C-ABI.

Names follow the reference (paths under subprojects/gst-plugins-base/):
  VideoInfo            ~ GstVideoInfo            gst-libs/gst/video/video-info.h:399
  VideoScaleMethod     ~ GstVideoScaleMethod     gst/videoconvertscale/gstvideoconvertscale.h:59
  CudaVideoConvertScale ~ the element: properties + GstVideoFilterClass::set_info /
                          ::transform_frame      gst/videoconvertscale/gstvideoconvertscale.c:906, :1981
The arithmetic lives in libb200dsp.so; this layer only marshals descriptors and pointers.
"""
import ctypes as C
import enum

import numpy as np

from . import _lib
from ._lib import lib, check


class VideoFormat(enum.IntEnum):
    I420 = 2
    YV12 = 3
    YUY2 = 4
    UYVY = 5
    Y42B = 18
    YVYU = 19
    Y444 = 20
    RGBx = 7
    BGRx = 8
    xRGB = 9
    xBGR = 10
    RGBA = 11
    BGRA = 12
    ARGB = 13
    ABGR = 14
    NV12 = 23
    # planar 8-bit RGB outputs: one byte plane per component (RGBP: R, G, B; BGRP: B, G, R).  A default-layout frame
    # whose width is a multiple of 4 is a contiguous (3, height, width) uint8 tensor.
    RGBP = 99
    BGRP = 100
    # compositor formats only (planar, little endian, 10 / 12 / 16 bits)
    I420_10LE = 43
    I422_10LE = 45
    Y444_10LE = 47
    I420_12LE = 73
    I422_12LE = 75
    Y444_12LE = 77
    Y444_16LE = 88
    NV21 = 24


class VideoScaleMethod(enum.IntEnum):
    NEAREST = 0
    BILINEAR = 1
    FOUR_TAP = 2
    LANCZOS = 3
    BILINEAR2 = 4
    SINC = 5
    HERMITE = 6
    SPLINE = 7
    CATROM = 8
    MITCHELL = 9


class ColorMatrix(enum.IntEnum):
    UNKNOWN = 0
    RGB = 1
    FCC = 2
    BT709 = 3
    BT601 = 4
    SMPTE240M = 5
    BT2020 = 6


class ColorRange(enum.IntEnum):
    UNKNOWN = 0
    RANGE_0_255 = 1
    RANGE_16_235 = 2


class ChromaSite(enum.IntFlag):
    UNKNOWN = 0
    NONE = 1
    H_COSITED = 2
    V_COSITED = 4
    ALT_LINE = 8
    COSITED = 6
    JPEG = 1
    MPEG2 = 2


def _ptr(x):
    """device/host pointer from an int, a torch tensor or a numpy array"""
    if x is None:
        return None
    if isinstance(x, int):
        return x
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    raise TypeError(f"cannot take a pointer from {type(x)}")


def _stream(s):
    if s is None:
        return None
    if isinstance(s, int):
        return s
    return s.cuda_stream  # torch.cuda.Stream


class VideoInfo:
    """Subset of GstVideoInfo the arithmetic depends on."""

    def __init__(self, fmt, width, height):
        self.c = _lib.VideoInfoC()
        check(lib.b200_video_info_set_format(C.byref(self.c), int(fmt), width, height),
              "b200_video_info_set_format")

    format = property(lambda s: VideoFormat(s.c.format))
    width = property(lambda s: s.c.width)
    height = property(lambda s: s.c.height)

    @property
    def size(self):
        return lib.b200_video_info_size(C.byref(self.c))

    @property
    def stride(self):
        return list(self.c.stride)

    @property
    def offset(self):
        return list(self.c.offset)

    def set_layout(self, strides, offsets):
        for i, (s, o) in enumerate(zip(strides, offsets)):
            self.c.stride[i] = s
            self.c.offset[i] = o
        return self

    def set_colorimetry(self, matrix=None, range=None, chroma_site=None):
        if matrix is not None:
            self.c.color_matrix = int(matrix)
        if range is not None:
            self.c.color_range = int(range)
        if chroma_site is not None:
            self.c.chroma_site = int(chroma_site)
        return self


_YUV_420 = (VideoFormat.I420, VideoFormat.YV12, VideoFormat.NV12, VideoFormat.NV21)
_YUV_422_PACKED = (VideoFormat.YUY2, VideoFormat.UYVY, VideoFormat.YVYU)


def transfer_colorimetry_from_input(in_info, out_info):
    """What the element's caps fixation does when the output caps leave colorimetry / chroma-site open
    (transfer_colorimetry_from_input, gstvideoconvertscale.c:1335-1427): a YUV output of a YUV input takes the input's
    colorimetry intact, and its chroma site too when the sub-sampling is unchanged (every format here is 4:2:0).
    RGB outputs keep their own defaults.  Returns out_info."""
    if in_info.format in _YUV_420 and out_info.format in _YUV_420:
        out_info.c.color_matrix = in_info.c.color_matrix
        out_info.c.color_range = in_info.c.color_range
        out_info.c.chroma_site = in_info.c.chroma_site
    elif in_info.format in _YUV_422_PACKED + (VideoFormat.Y42B, VideoFormat.Y444) and out_info.format in _YUV_420:
        # the sub-sampling changes: colorimetry carried over, chroma-site left to the output's own default (:1411-1424)
        out_info.c.color_matrix = in_info.c.color_matrix
        out_info.c.color_range = in_info.c.color_range
    return out_info


class PinnedBuffer:
    """Page-locked host staging buffer (b200_host_alloc), exposed as a numpy uint8 array."""

    def __init__(self, nbytes, device=None):
        p = C.c_void_p()
        if device is None:
            check(lib.b200_host_alloc(nbytes, C.byref(p)), "b200_host_alloc")
        else:                   # on the NUMA node that device hangs off
            check(lib.b200_host_alloc_near(device, nbytes, C.byref(p)), "b200_host_alloc_near")
        self.ptr = p.value
        self.nbytes = nbytes
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr))

    def free(self):
        if self.ptr:
            lib.b200_host_free(self.ptr)
            self.ptr = None
            self.array = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class CudaVideoConvertScale:
    """`cudavideoconvertscale`: same properties and call sequence as the stock element.

    method / envelope / sharpness / sharpen mirror the GObject properties
    (gstvideoconvertscale.c:306-391); `cuda_device_id` mirrors GstCudaBaseTransform's
    property (gst-plugins-bad/sys/nvcodec/gstcudabasetransform.c:89-90).
    """

    # the stock element's remaining properties and their defaults (gstvideoconvertscale.c:130-144, :306-391).  They are
    # accepted so that existing pipelines keep working; only the default of each is implemented (set_info refuses any
    # other value the way a failed converter setup does), and n-threads is free: the arithmetic is that of n-threads=1,
    # which differs from a multi-threaded reference run only in the chroma pairing at its slab boundaries (SURVEY A.4)
    REST_DEFAULTS = {"dither": "bayer", "dither_quantization": 1, "chroma_resampler": "linear", "alpha_mode": "copy",
                     "alpha_value": 1.0, "chroma_mode": "full", "matrix_mode": "full", "gamma_mode": "none",
                     "primaries_mode": "none", "converter_config": None}

    def __init__(self, method=VideoScaleMethod.BILINEAR, envelope=2.0, sharpness=1.0, sharpen=0.0,
                 cuda_device_id=0, add_borders=True, n_threads=1, **rest):
        unknown = set(rest) - set(self.REST_DEFAULTS)
        if unknown:
            raise TypeError(f"no such property: {sorted(unknown)}")
        self.n_threads = n_threads
        self.rest = dict(self.REST_DEFAULTS, **rest)
        # add-borders: TRUE like the stock element (DEFAULT_PROP_ADD_BORDERS, gstvideoconvertscale.c:131); the converter-level
        # parity tests pass add_borders=False (= gst_video_converter_new without a destination rectangle)
        self.add_borders = add_borders
        self.borders_w = self.borders_h = 0
        self.method = VideoScaleMethod(method)
        self.envelope = envelope
        self.sharpness = sharpness
        self.sharpen = sharpen
        self.cuda_device_id = cuda_device_id
        self._h = None
        self.in_info = self.out_info = None

    # GstVideoFilterClass::set_info
    def set_info(self, in_info, out_info):
        self._free()
        for k, v in self.rest.items():
            # dither only acts when quantising (8 -> 8 bit with dither-quantization 1 never does, video-converter.c:2056-2079)
            if k != "dither" and v != self.REST_DEFAULTS[k]:
                raise _lib.B200Error(-2, f"property {k.replace('_', '-')}={v!r}: only the default is implemented")
        cfg = _lib.VcsConfigC()
        lib.b200_vcs_config_init(C.byref(cfg))
        cfg.method = int(self.method)
        cfg.envelope, cfg.sharpness, cfg.sharpen = self.envelope, self.sharpness, self.sharpen
        # gst_video_convert_scale_set_info (gstvideoconvertscale.c:920-952): when the display aspect ratio changes (pixel
        # aspect ratio 1/1 on both sides here) and add-borders is set, scale into a centred rectangle that keeps it
        self.borders_w = self.borders_h = 0
        if self.add_borders:
            from math import gcd
            iw, ih, ow, oh = in_info.width, in_info.height, out_info.width, out_info.height
            g1, g2 = gcd(iw, ih), gcd(ow, oh)
            n, d = iw // g1, ih // g1
            if (n, d) != (ow // g2, oh // g2):
                to_h = ow * d // n
                if to_h <= oh:
                    self.borders_h = oh - to_h
                else:
                    self.borders_w = ow - oh * n // d
            cfg.dest_x, cfg.dest_y = self.borders_w // 2, self.borders_h // 2
            cfg.dest_width, cfg.dest_height = ow - self.borders_w, oh - self.borders_h
        h = C.c_void_p()
        check(lib.b200_vcs_create(C.byref(in_info.c), C.byref(out_info.c), C.byref(cfg),
                                  self.cuda_device_id, C.byref(h)), "b200_vcs_create")
        self._h = h
        self.in_info, self.out_info = in_info, out_info
        return True

    # GstVideoFilterClass::transform_frame — frames are device memory (GST_MAP_CUDA)
    def transform_frame(self, in_frame, out_frame, stream=None):
        check(lib.b200_vcs_convert(self._h, _ptr(in_frame), _ptr(out_frame), _stream(stream)),
              "b200_vcs_convert")

    def transform_frames(self, in_frames, out_frames, stream=None):
        n = len(in_frames)
        ins = (C.c_void_p * n)(*[_ptr(f) for f in in_frames])
        outs = (C.c_void_p * n)(*[_ptr(f) for f in out_frames])
        check(lib.b200_vcs_convert_batch(self._h, n, ins, outs, _stream(stream)),
              "b200_vcs_convert_batch")

    # system-memory peers: pinned staging + side streams inside the library
    def transform_host_frames(self, in_frames, out_frames):
        n = len(in_frames)
        ins = (C.c_void_p * n)(*[_ptr(f) for f in in_frames])
        outs = (C.c_void_p * n)(*[_ptr(f) for f in out_frames])
        check(lib.b200_vcs_convert_host(self._h, n, ins, outs), "b200_vcs_convert_host")

    def copy_probe(self, in_frames, out_frames):
        """the copies of transform_host_frames without the kernels (b200_vcs_copy_probe): the link's ceiling"""
        n = len(in_frames)
        ins = (C.c_void_p * n)(*[_ptr(f) for f in in_frames])
        outs = (C.c_void_p * n)(*[_ptr(f) for f in out_frames])
        check(lib.b200_vcs_copy_probe(self._h, n, ins, outs), "b200_vcs_copy_probe")

    # ---- introspection -------------------------------------------------------------
    def plan_info(self):
        info = _lib.VcsPlanInfoC()
        check(lib.b200_vcs_get_plan_info(self._h, C.byref(info)))
        return info

    def kernel_name(self):
        """the kernel (the first one of a multi-launch path) this plan runs: b200_vcs_kernel_name"""
        return lib.b200_vcs_kernel_name(self._h).decode()

    def matrix(self):
        im = (C.c_int32 * 16)()
        check(lib.b200_vcs_get_matrix(self._h, im))
        return np.array(list(im), dtype=np.int32).reshape(4, 4)

    def taps(self, direction):
        size = (self.out_info.width if direction == 0 else self.out_info.height)
        off = np.zeros(size, dtype=np.uint32)
        coef = np.zeros(size * 128, dtype=np.int16)
        per = check(lib.b200_vcs_get_taps(self._h, direction, off.ctypes.data, coef.ctypes.data,
                                          off.size, coef.size))
        return off, coef[:size * per].reshape(size, per) if per else coef[:0]

    def chroma_plan(self):
        m = np.zeros(self.in_info.height, dtype=np.uint8)
        check(lib.b200_vcs_get_chroma_plan(self._h, m.ctypes.data, m.size))
        return m

    def set_kernel_variant(self, v):
        check(lib.b200_vcs_set_kernel_variant(self._h, v), "b200_vcs_set_kernel_variant")

    def _free(self):
        if self._h:
            lib.b200_vcs_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass
