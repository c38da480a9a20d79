"""Host-side mirror of the reference compositor's interface over the C-ABI.

  CudaCompositor          ~ the `compositor` element: `background` property (compositor.c:742),
                            request sink pads, GstVideoAggregatorClass::aggregate_frames (:1739)
  CudaCompositorPad       ~ GstCompositorPad: xpos / ypos / width / height / alpha / operator / sizing-policy
                            (compositor.c:190-196, :678-716)
"""
import ctypes as C
import enum

from . import _lib
from ._lib import lib, check
from .video import VideoFormat, _ptr, _stream


class Background(enum.IntEnum):
    CHECKER = 0
    BLACK = 1
    WHITE = 2
    TRANSPARENT = 3


class Operator(enum.IntEnum):
    SOURCE = 0
    OVER = 1
    ADD = 2


def pad_output_size(src_w, src_h, pad_w, pad_h, sizing_policy="none", zero_size_is_unscaled=True):
    """_mixer_pad_get_output_size (compositor.c:289-417) for pixel aspect ratio 1/1 everywhere: the size a pad's picture
    takes in the output and the offset that centres it.  pad_w / pad_h are the pad's width / height properties (unset:
    the source size), sizing_policy "none" or "keep-aspect-ratio".  Returns (width, height, x_offset, y_offset)."""
    from math import gcd
    if zero_size_is_unscaled:
        pad_w = src_w if pad_w <= 0 else pad_w
        pad_h = src_h if pad_h <= 0 else pad_h
    else:
        pad_w = src_w if pad_w < 0 else pad_w
        pad_h = src_h if pad_h < 0 else pad_h
    if pad_w == 0 or pad_h == 0:
        return 0, 0, 0, 0
    if sizing_policy in ("none", 0):
        # the display-ratio round trip (gst_video_calculate_display_ratio, :330-352) is the identity at 1/1
        return pad_w, pad_h, 0, 0
    g1, g2 = gcd(src_w, src_h), gcd(pad_w, pad_h)
    num, den = src_w // g1, src_h // g1
    if (num, den) == (pad_w // g2, pad_h // g2):
        return pad_w, pad_h, 0, 0
    sh = pad_w * den // num                     # gst_util_uint64_scale_int (pad_width, den, num)
    if sh == 0:
        return 0, 0, 0, 0
    # gst_video_center_rect (gstvideosink.c:122-164), scaling: doubles, then truncation to int
    src_ratio, dst_ratio = pad_w / sh, pad_w / pad_h
    if src_ratio > dst_ratio:
        w, h = pad_w, int(pad_w / src_ratio)
        return w, h, 0, (pad_h - h) // 2
    if src_ratio < dst_ratio:
        w, h = int(pad_h * src_ratio), pad_h
        return w, h, (pad_w - w) // 2, 0
    return pad_w, pad_h, 0, 0


class CudaCompositorPad:
    """GstCompositorPad.  `width`/`height` are the pad properties (compositor.c:190-196): the size the
    pad's picture takes in the output.  `in_info` is the pad's caps: the pad is a GstVideoAggregatorConvertPad and its
    frames are converted to the aggregator's format, colorimetry and chroma site at width x height
    (gstvideoaggregator.c:479-570, :782-830) by a GstVideoConverter with DEFAULT options - cubic b = c = 1/3
    (video-converter.c:791, video-resampler.c:63-64), i.e. exactly cudavideoconvertscale method=mitchell - when that
    conversion differs from the caps.  The conversion runs inside b200_comp_blend_convert."""

    def __init__(self, width, height, stride=None, xpos=0, ypos=0, alpha=1.0, operator=Operator.OVER, in_info=None,
                 sizing_policy="none"):
        # sizing-policy (compositor.c:714): "keep-aspect-ratio" shrinks a converting pad's picture inside width x height
        # so that the source's display aspect ratio survives, centred by x_offset / y_offset
        self.x_offset = self.y_offset = 0
        self.sizing_policy = sizing_policy
        if in_info is not None:
            width, height, self.x_offset, self.y_offset = pad_output_size(in_info.width, in_info.height, width, height,
                                                                          sizing_policy)
        self.width, self.height = width, height
        self.stride = stride or width * 4
        self.xpos, self.ypos, self.alpha, self.operator = xpos, ypos, alpha, Operator(operator)
        self.frame = None          # the pad's frame (device memory)
        self.in_info = in_info

    def set_frame(self, frame):
        self.frame = frame
        return self

    def conversion_info(self, out_info):
        """gst_video_aggregator_convert_pad_create_conversion_info + gst_compositor_pad_create_conversion_info: the
        aggregator's format, colorimetry and chroma site at the pad's output size; None when that is the pad's caps"""
        from .video import VideoInfo
        if self.in_info is None:
            return None
        conv = VideoInfo(out_info.format, self.width, self.height)
        conv.set_colorimetry(out_info.c.color_matrix, out_info.c.color_range, out_info.c.chroma_site)
        a, b = self.in_info.c, conv.c
        same = (a.format, a.width, a.height, a.color_matrix, a.color_range, a.chroma_site) == \
            (b.format, b.width, b.height, b.color_matrix, b.color_range, b.chroma_site)
        return None if same else conv


class CudaCompositor:
    def __init__(self, out_format, width, height, background=Background.CHECKER, cuda_device_id=0):
        self.background = Background(background)
        self.width, self.height, self.format = width, height, VideoFormat(out_format)
        self.sinkpads = []
        self.device = cuda_device_id
        self._convs = {}           # one converter per distinct (pad caps, conversion info): pads that share it batch
        h = C.c_void_p()
        check(lib.b200_comp_create(int(out_format), width, height, cuda_device_id, C.byref(h)),
              "b200_comp_create")
        self._h = h

    def request_pad(self, *args, **kw):
        pad = CudaCompositorPad(*args, **kw)
        self.sinkpads.append(pad)
        return pad

    YUV_FORMATS = (VideoFormat.I420, VideoFormat.YV12, VideoFormat.NV12, VideoFormat.NV21, VideoFormat.Y444, VideoFormat.Y42B,
                   VideoFormat.I420_10LE, VideoFormat.I420_12LE, VideoFormat.I422_10LE, VideoFormat.I422_12LE,
                   VideoFormat.Y444_10LE, VideoFormat.Y444_12LE, VideoFormat.Y444_16LE)

    @staticmethod
    def _key(info):
        c = info.c
        return (c.format, c.width, c.height, tuple(c.stride), tuple(c.offset), c.color_matrix, c.color_range, c.chroma_site)

    def _converter(self, in_info, conv_info, used):
        from .video import CudaVideoConvertScale, VideoScaleMethod
        key = (self._key(in_info), self._key(conv_info))
        if key not in self._convs:
            conv = CudaVideoConvertScale(add_borders=False, method=VideoScaleMethod.MITCHELL, cuda_device_id=self.device)
            conv.set_info(in_info, conv_info)
            self._convs[key] = conv
        used[key] = self._convs[key]
        return self._convs[key]

    # GstVideoAggregatorClass::aggregate_frames (outbuf is device memory).  out_info: the output's plane layout and
    # colorimetry (default layout otherwise); out_stride: the row stride of a packed RGB output.
    def aggregate_frames(self, outbuf, out_stride=None, stream=None, out_info=None):
        from .video import VideoInfo
        if out_info is None:
            out_info = VideoInfo(self.format, self.width, self.height)
            if self.format not in self.YUV_FORMATS and out_stride:
                out_info.set_layout([out_stride], [0])
        pads = [p for p in self.sinkpads if p.frame is not None]
        arr = (_lib.CompPadConvertC * max(len(pads), 1))()
        used = {}
        for i, p in enumerate(pads):
            conv_info = p.conversion_info(out_info)
            if p.in_info is not None:
                info = p.in_info
            else:
                info = VideoInfo(self.format, p.width, p.height)
                if self.format not in self.YUV_FORMATS:
                    info.set_layout([p.stride], [0])
            arr[i].data = _ptr(p.frame)
            arr[i].info = info.c
            arr[i].conv = self._converter(info, conv_info, used)._h if conv_info is not None else None
            arr[i].xpos, arr[i].ypos, arr[i].alpha, arr[i].op = p.xpos + p.x_offset, p.ypos + p.y_offset, p.alpha, int(p.operator)
        check(lib.b200_comp_blend_convert(self._h, _ptr(outbuf), C.byref(out_info.c), int(self.background), arr, len(pads),
                                          _stream(stream)), "b200_comp_blend_convert")
        # a converter no pad uses any more (a pad's caps or size changed) is destroyed (its cudaFree waits for the call)
        self._convs = used

    # system-memory peers: pad frames and the output are HOST buffers (addresses); see b200_comp_blend_host_submit
    def aggregate_host_frames(self, out_ptr, pad_ptrs, out_stride=None, wait=True):
        pads = [p for p in self.sinkpads]
        arr = (_lib.CompPadC * max(len(pads), 1))()
        for i, (p, ptr) in enumerate(zip(pads, pad_ptrs)):
            arr[i].data = ptr
            arr[i].width, arr[i].height, arr[i].stride = p.width, p.height, p.stride
            arr[i].xpos, arr[i].ypos, arr[i].alpha, arr[i].op = p.xpos + p.x_offset, p.ypos + p.y_offset, p.alpha, int(p.operator)
        fn = lib.b200_comp_blend_host if wait else lib.b200_comp_blend_host_submit
        check(fn(self._h, out_ptr, out_stride or self.width * 4, int(self.background), arr, len(pads)), "b200_comp_blend_host")

    def aggregate_host_frames_yuv(self, out_ptr, pad_ptrs, out_info=None, wait=True):
        """system-memory peers of a planar / semi-planar YUV compositor (b200_comp_blend_yuv_host[_submit])"""
        from .video import VideoInfo
        out_info = out_info or VideoInfo(self.format, self.width, self.height)
        pads = [p for p in self.sinkpads]
        arr = (_lib.CompPadYuvC * max(len(pads), 1))()
        keep = []
        for i, (p, ptr) in enumerate(zip(pads, pad_ptrs)):
            info = p.in_info or VideoInfo(self.format, p.width, p.height)
            keep.append(info)
            arr[i].data = ptr
            arr[i].info = info.c
            arr[i].xpos, arr[i].ypos, arr[i].alpha, arr[i].op = p.xpos + p.x_offset, p.ypos + p.y_offset, p.alpha, int(p.operator)
        fn = lib.b200_comp_blend_yuv_host if wait else lib.b200_comp_blend_yuv_host_submit
        check(fn(self._h, out_ptr, C.byref(out_info.c), int(self.background), arr, len(pads)), "b200_comp_blend_yuv_host")

    def host_wait(self, keep_in_flight=0):
        check(lib.b200_comp_blend_host_wait(self._h, keep_in_flight), "b200_comp_blend_host_wait")

    def __del__(self):
        try:
            if self._h:
                lib.b200_comp_destroy(self._h)
                self._h = None
        except Exception:
            pass
