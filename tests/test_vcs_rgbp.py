"""Planar RGB outputs (RGBP / BGRP) without a GPU: host plans, the frame layout, the oracle against the reference build,
the golden fixture, and the product's kernels under the CPU emulation (tests/cudaemu) against the oracle.

RGBP / BGRP take the reference's packed-RGB chain (pack_RGBP / pack_BGRP through ARGB): the same matrix, taps, pass
order and chroma pairing as BGRx, except that I420 / YV12 at an unchanged size has no convert_I420_BGRA-style table row
and so keeps its chroma up-sampling.  Packed RGB inputs run the matrix-free chain and a de-interleave."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

from oracle import bindings as ob
from rgbp_oracle import FMT, default_layout, frame_size, oracle_rgbp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tests", "cudaemu"))

YUV420 = ["NV12", "NV21", "I420", "YV12"]
RGB = ["BGRA", "RGBA", "ARGB", "ABGR", "BGRx", "RGBx", "xRGB", "xBGR"]
CAPTURE = ["YUY2", "UYVY", "YVYU", "Y42B", "Y444"]
SINKS = YUV420 + RGB + CAPTURE
OUTS = ["RGBP", "BGRP"]


def frame_for(fmt, iw, ih, seed):
    d = ob.vcs_desc(iw, ih, iw, ih, 1, in_fmt=FMT[fmt], out_fmt=12)
    return np.random.default_rng(seed).integers(0, 256, ob.vcs_sizes(d)[0], dtype=np.uint8)


oracle_out = oracle_rgbp


class Handle:
    """b200_vcs_create through the given library (the product with device -1, or the emulation with device 0)"""

    def __init__(self, lib, fi, fo, size, method, device, site=None, layout=None, dest=None, border=0xff000000,
                 matrix=None, rng=None):
        from gstreamer_b200 import _lib
        iw, ih, ow, oh = size
        self.lib = lib
        self.ii, self.oi = _lib.VideoInfoC(), _lib.VideoInfoC()
        assert lib.b200_video_info_set_format(C.byref(self.ii), FMT[fi], iw, ih) == 0
        assert lib.b200_video_info_set_format(C.byref(self.oi), FMT[fo], ow, oh) == 0
        if site is not None:
            self.ii.chroma_site = site
        if matrix is not None:
            self.ii.color_matrix = matrix
        if rng is not None:
            self.ii.color_range = rng
        if layout:
            for k in range(3):
                self.oi.stride[k], self.oi.offset[k] = layout[0][k], layout[1][k]
        cfg = _lib.VcsConfigC()
        lib.b200_vcs_config_init(C.byref(cfg))
        cfg.method = method
        if dest:
            cfg.dest_x, cfg.dest_y, cfg.dest_width, cfg.dest_height = dest
            cfg.border_argb = border
        self.h = C.c_void_p()
        st = lib.b200_vcs_create(C.byref(self.ii), C.byref(self.oi), C.byref(cfg), device, C.byref(self.h))
        assert st == 0, (st, fi, fo, size)

    def info(self):
        from gstreamer_b200 import _lib
        i = _lib.VcsPlanInfoC()
        assert self.lib.b200_vcs_get_plan_info(self.h, C.byref(i)) == 0
        return i

    def convert(self, frame):
        out = np.full(self.lib.b200_video_info_size(C.byref(self.oi)), 0x5A, dtype=np.uint8)
        src = np.ascontiguousarray(frame)
        assert self.lib.b200_vcs_convert(self.h, src.ctypes.data, out.ctypes.data, None) == 0
        return out

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.lib.b200_vcs_destroy(self.h)


def check(got, want, tag):
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{tag}: {len(bad)} of {got.size} bytes differ, first at {bad[:5].ravel().tolist()}"


def product():
    from gstreamer_b200 import _lib
    return _lib.lib


# ---- 1. host plans (device -1) ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("fi,size,method,site,variant", [
    ("NV12", (512, 248, 256, 124), 3, 2, 1),       # exact 2:1, 8 taps: vcs_lanczos2_v2_kernel
    ("I420", (512, 248, 256, 124), 3, 2, 1),
    ("NV12", (1920, 1080, 1280, 720), 1, 2, 2),    # bilinear: vcs_light_kernel
    ("NV12", (1920, 1080, 640, 640), 3, 2, 3),     # anamorphic lanczos: vcs_ntap_kernel
    ("YUY2", (64, 48, 32, 24), 3, 2, 0),           # 4:2:2: vcs_generic_kernel
], ids=["l2-nv12", "l2-i420", "light", "ntap", "422"])
def test_plan_kernel_and_tables_equal_bgrx(fi, fo, size, method, site, variant):
    lib = product()
    with Handle(lib, fi, fo, size, method, -1, site=site) as p, Handle(lib, fi, "BGRx", size, method, -1, site=site) as q:
        a, b = p.info(), q.info()
        assert a.kernel_variant == variant == b.kernel_variant
        assert a.n_launches_per_convert == b.n_launches_per_convert == 1
        for f in ("h_taps", "v_taps", "h_first", "matrix_first", "tile_w", "tile_h", "smem_bytes"):
            assert getattr(a, f) == getattr(b, f), f
        assert list(a.p) == list(b.p)
        ma, mb = (C.c_int32 * 16)(), (C.c_int32 * 16)()
        lib.b200_vcs_get_matrix(p.h, ma)
        lib.b200_vcs_get_matrix(q.h, mb)
        assert list(ma) == list(mb) and any(ma)
        for d, n in ((0, size[2]), (1, size[3])):
            oa, ob_ = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
            ta, tb = np.zeros(n * 128, np.int16), np.zeros(n * 128, np.int16)
            assert lib.b200_vcs_get_taps(p.h, d, oa.ctypes.data, ta.ctypes.data, n, ta.size) == \
                lib.b200_vcs_get_taps(q.h, d, ob_.ctypes.data, tb.ctypes.data, n, tb.size)
            assert np.array_equal(oa, ob_) and np.array_equal(ta, tb)
        ca, cb = np.zeros(size[1], np.uint8), np.zeros(size[1], np.uint8)
        lib.b200_vcs_get_chroma_plan(p.h, ca.ctypes.data, ca.size)
        lib.b200_vcs_get_chroma_plan(q.h, cb.ctypes.data, cb.size)
        assert np.array_equal(ca, cb)


@pytest.mark.parametrize("fi", ["I420", "YV12"])
@pytest.mark.parametrize("fo", OUTS)
def test_i420_same_size_keeps_chroma_upsampling(fi, fo):
    """I420 -> BGRx at an unchanged size is the convert_I420_BGRA table row (nearest chroma: every line mode 0); planar
    RGB has no such row, so its lines pair up for the vertical chroma filter like any scaled plan"""
    lib = product()
    size = (64, 48, 64, 48)
    with Handle(lib, fi, fo, size, 1, -1) as p, Handle(lib, fi, "BGRx", size, 1, -1) as q:
        ca, cb = np.zeros(48, np.uint8), np.zeros(48, np.uint8)
        lib.b200_vcs_get_chroma_plan(p.h, ca.ctypes.data, 48)
        lib.b200_vcs_get_chroma_plan(q.h, cb.ctypes.data, 48)
        assert not cb.any(), "packed RGB: nearest chroma"
        assert ca.tolist() == [0] + [1 if y & 1 else 2 for y in range(1, 48)], "planar RGB: standard line pairs"
    frame = ob.i420_random_frame(64, 48, 3)
    d_rgbp = oracle_out(fi, fo, size, 1, frame)
    d_bgrx = ob.oracle_vcs_convert(ob.vcs_desc(64, 48, 64, 48, 1, in_fmt=FMT[fi], out_fmt=FMT["BGRx"]), frame).reshape(48, 64, 4)
    # bytes differ from a de-interleaved BGRx frame: the filtered chroma is not the replicated one
    planes = d_rgbp.reshape(3, 48, 64)
    assert not np.array_equal(planes[1], d_bgrx[:, :, 1])


@pytest.mark.parametrize("fi", ["BGRA", "xRGB", "ABGR"])
@pytest.mark.parametrize("fo", OUTS)
def test_packed_rgb_route(fi, fo):
    lib = product()
    for size, launches in (((64, 48, 64, 48), 1), ((64, 48, 40, 30), 2), ((40, 30, 64, 48), 2)):
        with Handle(lib, fi, fo, size, 3, -1) as p:
            i = p.info()
            assert i.kernel_variant == 4 and i.n_launches_per_convert == launches, (size, i.n_launches_per_convert)
            assert lib.b200_vcs_kernel_name(p.h) == b"vcs_rgb_deinterleave_kernel"
            m = (C.c_int32 * 16)()
            lib.b200_vcs_get_matrix(p.h, m)
            assert not any(m), "no matrix stage"
    with Handle(lib, fi, fo, (64, 48, 40, 30), 3, -1, dest=(4, 2, 30, 20)) as p:
        assert p.info().n_launches_per_convert == 3          # border fill + scaler + de-interleave


@pytest.mark.parametrize("fo", OUTS)
def test_strides_below_width_refused(fo):
    from gstreamer_b200 import _lib
    lib = product()
    for fi in ("NV12", "BGRA"):
        ii, oi = _lib.VideoInfoC(), _lib.VideoInfoC()
        lib.b200_video_info_set_format(C.byref(ii), FMT[fi], 64, 48)
        lib.b200_video_info_set_format(C.byref(oi), FMT[fo], 64, 48)
        oi.stride[2] = 63
        h = C.c_void_p()
        assert lib.b200_vcs_create(C.byref(ii), C.byref(oi), None, -1, C.byref(h)) == -1


# ---- 2. layout ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("w,h", [(1, 1), (2, 3), (5, 7), (64, 48), (1919, 1081), (1920, 1080)])
def test_video_info_layout(fo, w, h):
    import gstreamer_b200 as g
    vi = g.VideoInfo(FMT[fo], w, h)
    s = (w + 3) & ~3
    assert vi.stride[:3] == [s, s, s] and vi.offset[:3] == [0, s * h, 2 * s * h] and vi.size == 3 * s * h
    assert vi.c.color_matrix == 1 and vi.c.color_range == 1


@pytest.mark.ref
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("w,h", [(1, 1), (2, 3), (5, 7), (64, 48), (1919, 1081), (1920, 1080)])
def test_video_info_layout_matches_reference(fo, w, h):
    import gstreamer_b200 as g
    r = ob.ref()
    r.ref_video_info.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int * 4),
                                 C.POINTER(C.c_size_t * 4), C.POINTER(C.c_size_t)]
    n, st, off, size = C.c_int(), (C.c_int * 4)(), (C.c_size_t * 4)(), C.c_size_t()
    assert r.ref_video_info(FMT[fo], w, h, C.byref(n), C.byref(st), C.byref(off), C.byref(size)) == 0
    vi = g.VideoInfo(FMT[fo], w, h)
    assert n.value == 3 and vi.stride[:3] == list(st)[:3] and vi.offset[:3] == list(off)[:3] and vi.size == size.value


# ---- 3. the expected bytes (tests/rgbp_oracle.py: the oracle's packed chain, de-interleaved) against the reference build ---
ORACLE_SIZES = [(1, 1, 1, 1), (7, 5, 3, 9), (33, 17, 20, 31), (64, 48, 64, 48), (65, 49, 65, 49), (40, 30, 64, 48), (2, 3, 1, 1)]


def _ref_out(fi, fo, size, method, frame, site=-1, matrix=-1, rng=-1, dest=None, border=None):
    iw, ih, ow, oh = size
    r = ob.RefVcs(iw, ih, ow, oh, method, in_fmt=FMT[fi], out_fmt=FMT[fo], site=site, matrix=matrix, rng=rng,
                  dest=dest, border_argb=border)
    out = r.convert(frame, np.full(frame_size(default_layout(ow, oh), oh), 0x5A, dtype=np.uint8))
    r.close()
    return out


@pytest.mark.ref
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("fi", SINKS)
def test_oracle_matches_reference(fi, fo):
    for size in ORACLE_SIZES:
        for m in range(10):
            frame = frame_for(fi, size[0], size[1], m + size[0])
            check(oracle_out(fi, fo, size, m, frame), _ref_out(fi, fo, size, m, frame), f"{fi}->{fo} {size} m{m}")


@pytest.mark.ref
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("fi", YUV420 + CAPTURE)
@pytest.mark.parametrize("matrix", [4, 3, 6], ids=["bt601", "bt709", "bt2020"])
@pytest.mark.parametrize("rng", [1, 2], ids=["full", "limited"])
def test_oracle_colorimetry_matches_reference(fi, fo, matrix, rng):
    for size, m, site in (((64, 48, 40, 30), 3, 2), ((33, 17, 33, 17), 1, 1), ((20, 12, 50, 31), 9, 2)):
        frame = frame_for(fi, size[0], size[1], matrix * 10 + rng)
        check(oracle_out(fi, fo, size, m, frame, site=site, matrix=matrix, rng=rng),
              _ref_out(fi, fo, size, m, frame, site=site, matrix=matrix, rng=rng), f"{fi}->{fo} {size} m{m}")


@pytest.mark.ref
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("fi", ["NV12", "I420", "BGRA", "YUY2"])
@pytest.mark.parametrize("border", [0xff000000, 0x80ff4010, 0x00123456])
def test_oracle_borders_match_reference(fi, fo, border):
    for size in ((64, 48, 64, 36), (48, 48, 40, 30), (33, 17, 20, 31)):
        dest = ob.vcs_borders(*size)
        frame = frame_for(fi, size[0], size[1], 7)
        check(oracle_out(fi, fo, size, 3, frame, dest=dest, border=border),
              _ref_out(fi, fo, size, 3, frame, dest=dest, border=border), f"{fi}->{fo} {size} {dest}")


def test_golden_fixture():
    arrays = np.load(os.path.join(GOLDEN, "video_rgbp.npz"))
    cases = json.load(open(os.path.join(GOLDEN, "video_rgbp_cases.json")))
    assert len(cases) >= 100
    for c in cases:
        (iw, ih), (ow, oh) = c["in"], c["out"]
        frame = frame_for(c["in_fmt"], iw, ih, c["seed"])
        check(oracle_rgbp(c["in_fmt"], c["out_fmt"], (iw, ih, ow, oh), c["method"], frame, site=c["site"], fill=0),
              arrays[c["key"]], c["key"])


# ---- 4. the product's kernels under the CPU emulation ---------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    import build_emu
    from gstreamer_b200 import _lib
    lib = C.CDLL(build_emu.build())
    for name, (res, args) in _lib._SIGS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return lib


def _odd_layout(ow, oh, order=(2, 0, 1)):
    """plane strides above the width, unaligned offsets, planes in memory in `order`"""
    strides = [ow + 5, ow + 3, ow + 9]
    offs, pos = [0, 0, 0], 3
    for k in order:
        offs[k] = pos
        pos += strides[k] * oh + 7
    return strides, offs


EMU_CASES = [
    ("NV12", (512, 248, 256, 124), 3, 2, 1), ("I420", (512, 248, 256, 124), 9, 2, 1),      # 2:1 lanczos, second form
    ("NV12", (64, 48, 40, 30), 1, 2, 2), ("NV21", (100, 60, 150, 30), 1, 1, 2),           # light: h first / v first
    ("I420", (64, 48, 64, 48), 1, 1, 2),                                                  # light, same-size I420 (chain)
    ("NV12", (96, 54, 64, 36), 3, 2, 3), ("NV12", (100, 60, 150, 30), 3, 2, 3),          # n-tap: h first / v first
    ("YV12", (64, 48, 40, 30), 9, 1, 3),
    ("YUY2", (33, 17, 20, 31), 3, 2, 0), ("Y42B", (40, 30, 64, 48), 1, 1, 0), ("Y444", (33, 17, 33, 17), 9, 2, 0),
]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("case", EMU_CASES, ids=lambda c: "%s-%dx%d-%dx%d-m%d-v%d" % (c[0], *c[1], c[2], c[4]))
def test_emulated_kernels(emu, case, fo):
    fi, size, method, site, variant = case
    frame = frame_for(fi, size[0], size[1], 11)
    want = oracle_out(fi, fo, size, method, frame, site=site)
    with Handle(emu, fi, fo, size, method, 0, site=site) as p:
        assert p.info().kernel_variant == variant
        check(p.convert(frame), want, f"{fi}->{fo} v{variant}")
        if variant:
            assert emu.b200_vcs_set_kernel_variant(p.h, 0) == 0
            check(p.convert(frame), want, f"{fi}->{fo} generic")
        if variant == 1:            # the first form and the tensor forms decline planar output
            assert emu.b200_vcs_set_kernel_variant(p.h, 6) == -2
            assert emu.b200_vcs_set_kernel_variant(p.h, 7) == -2
    layout = _odd_layout(size[2], size[3])
    want = oracle_out(fi, fo, size, method, frame, site=site, layout=layout)
    with Handle(emu, fi, fo, size, method, 0, site=site, layout=layout) as p:
        assert p.info().kernel_variant == variant, "plane layouts do not change the kernel"
        check(p.convert(frame), want, f"{fi}->{fo} v{variant} odd layout")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("fi", ["NV12", "I420", "BGRA", "YUY2"])
def test_emulated_borders(emu, fi, fo):
    for size, border in (((64, 48, 64, 36), 0x80ff4010), ((48, 48, 40, 30), 0x00123456)):
        dest = ob.vcs_borders(*size)
        frame = frame_for(fi, size[0], size[1], 5)
        want = oracle_out(fi, fo, size, 3, frame, site=2 if fi not in RGB else None, dest=dest, border=border)
        with Handle(emu, fi, fo, size, 3, 0, site=2 if fi not in RGB else None, dest=dest, border=border) as p:
            check(p.convert(frame), want, f"{fi}->{fo} {size} dest {dest}")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("fi", RGB)
def test_emulated_packed_rgb(emu, fi, fo):
    for size in ((40, 30, 40, 30), (33, 17, 20, 31), (40, 30, 64, 48), (7, 5, 3, 9)):
        for m in (0, 1, 3):
            frame = frame_for(fi, size[0], size[1], m)
            check(_emu_convert(emu, fi, fo, size, m, frame), oracle_out(fi, fo, size, m, frame), f"{fi}->{fo} {size} m{m}")
    layout = _odd_layout(20, 31, (1, 2, 0))
    frame = frame_for(fi, 33, 17, 9)
    with Handle(emu, fi, fo, (33, 17, 20, 31), 3, 0, layout=layout) as p:
        check(p.convert(frame), oracle_out(fi, fo, (33, 17, 20, 31), 3, frame, layout=layout), "odd layout")


def _emu_convert(emu, fi, fo, size, m, frame):
    with Handle(emu, fi, fo, size, m, 0) as p:
        return p.convert(frame)
