"""b200_comp_blend_convert (convert pads) through the emulated library (tests/cudaemu): every output byte against the
expected bytes of existing code only - each converted pad through oracle_vcs_convert (method mitchell, the output's
colorimetry, the pad's output size), then oracle_compositor / oracle_compositor_yuv - and the route each pad takes, read
from the emulator's launch log."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle import bindings as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "cudaemu"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.timeout(900)

import comp_convert_cases as cc  # noqa: E402


@pytest.fixture(scope="module")
def emu():
    import build_emu
    from gstreamer_b200 import _lib
    lib = C.CDLL(build_emu.build())
    for name, (res, args) in _lib._SIGS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    lib.b200emu_set_record_only.argtypes = [C.c_int]
    lib.b200emu_launch_log.restype = C.c_char_p
    return lib


class EmuMem:
    """'device memory' of the emulated library: host arrays"""

    def __init__(self):
        self.keep = []

    def upload(self, a):
        a = np.ascontiguousarray(a)
        self.keep.append(a)
        return a.ctypes.data, a

    def download(self, handle):
        return handle.copy()


@pytest.mark.parametrize("out_name", ["I420", "YV12", "NV12", "NV21", "BGRA", "RGBA", "ARGB", "ABGR"])
def test_random_layouts(emu, out_name):
    """random layouts: pads in NV12 / NV21 / I420 / YV12 / YUY2 / Y444 / BGRx that grow and shrink (odd sizes too), hang
    off every edge at odd positions, every alpha class, operator and background, fused and blend-kernel pads interleaved
    and overlapping, keep-aspect-ratio offsets, shared converters, odd plane strides and offsets"""
    rng = np.random.default_rng(cc.FMT[out_name])
    for trial in range(4):
        case = cc.random_case(rng, out_name, trial, max_size=(56, 40), max_pads=6 if trial < 3 else 9)
        got, want, routes = cc.run_case(emu, EmuMem(), case, None, log=emu)
        cc.check_bytes(got, want, f"{out_name} trial {trial}")
        cc.check_routes(case, routes)


def test_many_pads(emu):
    """more than 32 pads (two blend-kernel chunks and fused groups between them)"""
    rng = np.random.default_rng(5)
    case = cc.random_case(rng, "NV12", 0, max_size=(48, 32), max_pads=40, min_pads=40, pad_max=(12, 10))
    got, want, routes = cc.run_case(emu, EmuMem(), case, None, log=emu)
    cc.check_bytes(got, want, "40 pads")
    cc.check_routes(case, routes)


@pytest.mark.parametrize("out_name", ["NV12", "I420"])
def test_mosaic_route(emu, out_name):
    """a 4 x 4 mosaic of tiles sharing one converter: one background launch plus the plane scalers of one converter
    group (one launch per plane kernel), no converted frame; then the same with one blended pad on top"""
    case = cc.mosaic_case(out_name, tile=(16, 10), src=(32, 20), grid=(4, 4))
    log = cc.route_log(emu, case)
    n_scaler = len(log) - 1
    assert log[0] == "comp_yuv_kernel", log
    assert all("_comp_kernel" in k for k in log[1:]), log
    assert 2 <= len(log) <= 1 + cc.conv_launches(emu, case), log          # copy / halve planes share the byte kernel's launch
    got, want, routes = cc.run_case(emu, EmuMem(), case, None, log=emu)
    cc.check_bytes(got, want, "mosaic")
    case["pads"].append(dict(case["pads"][0], x=5, y=3, alpha=0.5))
    got, want, routes = cc.run_case(emu, EmuMem(), case, None, log=emu)
    cc.check_bytes(got, want, "mosaic + overlay")
    log = cc.route_log(emu, case)
    assert sum("_comp_kernel" in k for k in log) == 2 * n_scaler, log


def test_alpha_zero_pads_are_not_converted(emu):
    case = cc.mosaic_case("BGRA", tile=(16, 10), src=(32, 20), grid=(2, 1))
    for p in case["pads"]:
        p["alpha"] = 0.0
    log = cc.route_log(emu, case)
    assert log == ["comp_kernel"], log
