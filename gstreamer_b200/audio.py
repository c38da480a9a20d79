"""Host-side mirror of the reference audioresample interface over the C-ABI.

  CudaAudioResample ~ the `audioresample` element: `quality` property (gstaudioresample.c:68),
                      set_caps -> resampler setup (:398-460), transform (:885-957),
                      reset on flush/discont (:462, :907-915), drain (:590-662)
The arithmetic (filter design on the host, polyphase FIR on the device) lives in libb200dsp.so.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import lib, check, B200Error
from .video import _ptr, _stream


class AudioFormat:
    """GstAudioFormat values of every interleaved sample format the element resamples.  S16LE, S32LE, F32LE and F64LE are
    resampled as they are (audio-converter.c:700-727); the others are unpacked to S32 or F64 inside the kernels and
    quantized and packed back on store."""
    S8, U8, S16LE, S16BE, U16LE, U16BE = 2, 3, 4, 5, 6, 7
    S24_32LE, S24_32BE, U24_32LE, U24_32BE, S32LE, S32BE, U32LE, U32BE = 8, 9, 10, 11, 12, 13, 14, 15
    S24LE, S24BE, U24LE, U24BE, S20LE, S20BE, U20LE, U20BE, S18LE, S18BE, U18LE, U18BE = range(16, 28)
    F32LE, F32BE, F64LE, F64BE = 28, 29, 30, 31
    S20_32LE, S20_32BE, U20_32LE, U20_32BE = 32, 33, 34, 35
    DTYPE = {4: np.int16, 12: np.int32, 28: np.float32, 30: np.float64}
    # bytes per sample in a buffer (GST_AUDIO_FORMAT_INFO_WIDTH / 8)
    WIDTH = {2: 1, 3: 1, 4: 2, 5: 2, 6: 2, 7: 2, **{v: 4 for v in range(8, 16)}, **{v: 3 for v in range(16, 28)},
             28: 4, 29: 4, 30: 8, 31: 8, 32: 4, 33: 4, 34: 4, 35: 4}
    NAMES = {2: "S8", 3: "U8", 4: "S16LE", 5: "S16BE", 6: "U16LE", 7: "U16BE", 8: "S24_32LE", 9: "S24_32BE", 10: "U24_32LE",
             11: "U24_32BE", 12: "S32LE", 13: "S32BE", 14: "U32LE", 15: "U32BE", 16: "S24LE", 17: "S24BE", 18: "U24LE",
             19: "U24BE", 20: "S20LE", 21: "S20BE", 22: "U20LE", 23: "U20BE", 24: "S18LE", 25: "S18BE", 26: "U18LE",
             27: "U18BE", 28: "F32LE", 29: "F32BE", 30: "F64LE", 31: "F64BE", 32: "S20_32LE", 33: "S20_32BE",
             34: "U20_32LE", 35: "U20_32BE"}


class CudaAudioResample:
    # the stock element's remaining properties (gstaudioresample.c:153-186) with their nicks.  Implemented: both
    # windowed-sinc methods, every filter mode, every table interpolation, and the nearest / linear / cubic methods
    # (device-verified: tests/test_ars_options_gpu.py).
    # sinc-filter-auto-threshold never reaches the reference's resampler (UINT stored, INT read: SURVEY A.10)
    REST_DEFAULTS = {"resample_method": "kaiser", "sinc_filter_mode": "auto", "sinc_filter_interpolation": "cubic"}
    METHODS = {"nearest": 1, "linear": 2, "cubic": 3, "blackman-nuttall": 4, "kaiser": 5}
    FILTER_MODES = {"interpolated": 1, "full": 2, "auto": 3}
    INTERPOLATIONS = {"none": 1, "linear": 2, "cubic": 3}

    def __init__(self, quality=4, cuda_device_id=0, format=AudioFormat.F32LE, sinc_filter_auto_threshold=1048576, **rest):
        unknown = set(rest) - set(self.REST_DEFAULTS)
        if unknown:
            raise TypeError(f"no such property: {sorted(unknown)}")
        self.rest = dict(self.REST_DEFAULTS, **rest)
        self.sinc_filter_auto_threshold = sinc_filter_auto_threshold
        self.quality = quality
        self.format = format
        self.cuda_device_id = cuda_device_id
        self._h = None
        self.passthrough = False
        self.in_rate = self.out_rate = self.channels = None

    # GstBaseTransformClass::set_caps (interleaved samples of self.format)
    def set_caps(self, in_rate, out_rate, channels):
        # gst_audio_resample_update_state (gstaudioresample.c:398-437): same format and channel count on a live resampler
        # = a rate change, the converter is UPDATED (history and phase survive); anything else builds a new one
        if self._h is not None and channels == getattr(self, "channels", None) and in_rate != out_rate:
            self.update_rates(in_rate, out_rate)
            self.in_rate, self.out_rate = in_rate, out_rate
            return True
        self._free()
        # gst_audio_resample_set_caps: equal rates put the base transform in pass-through mode (buffers are forwarded
        # untouched and transform() is never called)
        self.passthrough = in_rate == out_rate
        if self.passthrough:
            self.in_rate, self.out_rate, self.channels = in_rate, out_rate, channels
            return True
        method = self.METHODS[self.rest["resample_method"]]
        mode = self.FILTER_MODES[self.rest["sinc_filter_mode"]]
        interp = self.INTERPOLATIONS[self.rest["sinc_filter_interpolation"]]
        cfg = _lib.ArsConfigC()
        cfg.in_rate, cfg.out_rate, cfg.channels, cfg.quality = in_rate, out_rate, channels, self.quality
        cfg.format = int(self.format)
        cfg.resample_method, cfg.sinc_filter_mode, cfg.sinc_filter_interpolation = method, mode, interp
        h = C.c_void_p()
        check(lib.b200_ars_create(C.byref(cfg), self.cuda_device_id, C.byref(h)), "b200_ars_create")
        self._h = h
        self.in_rate, self.out_rate, self.channels = in_rate, out_rate, channels
        return True

    def get_out_frames(self, in_frames):
        return lib.b200_ars_get_out_frames(self._h, in_frames)

    def get_in_frames(self, out_frames):
        return lib.b200_ars_get_in_frames(self._h, out_frames)

    @property
    def max_latency(self):
        return lib.b200_ars_get_max_latency(self._h)

    # GstBaseTransformClass::transform — device buffers, F32 interleaved; inbuf None = drain zeros
    def transform(self, inbuf, in_frames, outbuf, out_capacity, stream=None):
        if self._h is None:
            raise B200Error(-1, "transform() in pass-through mode (equal rates): the buffer is forwarded as it is")
        n = C.c_size_t()
        check(lib.b200_ars_process(self._h, _ptr(inbuf), in_frames, _ptr(outbuf), out_capacity, C.byref(n),
                                   _stream(stream)), "b200_ars_process")
        return n.value

    # system-memory peers: host buffers in, host buffers out (pinned ring + side streams inside the library)
    def transform_host(self, in_ptr, in_frames, out_ptr, out_capacity, wait=True):
        """wait=False: queued (b200_ars_process_host_submit); host_wait(k) later returns when all but the k latest are done"""
        n = C.c_size_t()
        fn = lib.b200_ars_process_host if wait else lib.b200_ars_process_host_submit
        check(fn(self._h, in_ptr, in_frames, out_ptr, out_capacity, C.byref(n)), "b200_ars_process_host")
        return n.value

    def host_wait(self, keep_in_flight=0):
        check(lib.b200_ars_process_host_wait(self._h, keep_in_flight), "b200_ars_process_host_wait")

    def reset(self):
        check(lib.b200_ars_reset(self._h), "b200_ars_reset")

    def update_rates(self, in_rate, out_rate):
        """new caps with the same format / channels on a live stream (gst_audio_resample_update_state): keeps history"""
        check(lib.b200_ars_update(self._h, in_rate, out_rate), "b200_ars_update")

    def plan_info(self):
        info = _lib.ArsPlanInfoC()
        check(lib.b200_ars_get_plan_info(self._h, C.byref(info)))
        return info

    def phase_taps(self, phase):
        n = self.plan_info().n_taps
        t = np.zeros(n, dtype=np.float32)
        check(lib.b200_ars_get_phase_taps(self._h, phase, t.ctypes.data, n))
        return t

    def _free(self):
        if self._h:
            lib.b200_ars_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass
