"""gstreamer_b200 — CUDA-native (H100, sm_90a) raw-frame DSP hot path behind GStreamer's element surface.

Python is the test/bench harness and the host-side mirror of the reference's element
interface; the product is gstreamer_b200/libb200dsp.so (hand-written sm_90a CUDA +
C-ABI, include/b200dsp.h).  Importing this package without the built library fails.
"""
from ._lib import lib, LIB_PATH, B200Error, EXPORTED_SYMBOLS, MISSING_SYMBOLS  # noqa: F401
from .video import (VideoFormat, VideoScaleMethod, ColorMatrix, ColorRange, ChromaSite,  # noqa: F401
                    VideoInfo, PinnedBuffer, CudaVideoConvertScale, transfer_colorimetry_from_input)

__all__ = ["lib", "LIB_PATH", "B200Error", "VideoFormat", "VideoScaleMethod", "ColorMatrix",
           "ColorRange", "ChromaSite", "VideoInfo", "PinnedBuffer", "CudaVideoConvertScale", "transfer_colorimetry_from_input"]
