"""Packed RGB -> 4:2:0 (BGRA -> NV12 ...: what sits between a compositor and an encoder).  The reference runs its
generic chain: unpack to ARGB, the scalers that shrink, the RGB -> YUV table matrix (video_converter_matrix8_table,
video-converter.c:1178-1200), the scalers that grow, chroma down-sampling, 4:2:0 pack.  Product: vcs_generic_kernel
(packed-pixel input stage, matrix between the passes) into scratch A,Y,U,V images, then vcs_down420_kernel.

Packed RGB -> packed RGB takes the plane-scaling fast path (convert_scale_planes): vcs_planes_fast_kernel on 4-byte
pixels where the shape is eligible, the byte-wise vcs_planes_kernel otherwise."""
import os

import numpy as np
import pytest

from oracle import bindings as ob

pytestmark = [pytest.mark.gpu]

RGB_IN = ["BGRA", "RGBA", "ARGB", "ABGR", "BGRx", "RGBx", "xRGB", "xBGR"]
YUV_OUT = ["NV12", "I420", "NV21", "YV12"]
SIZES = [(64, 48, 32, 24), (64, 48, 96, 72), (65, 49, 33, 26), (33, 17, 20, 31), (50, 21, 50, 21), (57, 35, 29, 35),
         (100, 100, 150, 50), (40, 90, 40, 31), (17, 9, 64, 31), (2, 2, 1, 1), (1, 1, 5, 4), (640, 480, 320, 240),
         (1920, 1080, 1280, 720), (1280, 720, 1920, 1080)]


def rgb_frame(iw, ih, seed):
    return np.random.default_rng(seed).integers(0, 256, iw * ih * 4, dtype=np.uint8)


def convert(size, method, frame, fi, fo, colorimetry=None):
    import torch
    import gstreamer_b200 as g
    iw, ih, ow, oh = size
    el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
    ii, oi = g.VideoInfo(ob.FMT[fi], iw, ih), g.VideoInfo(ob.FMT[fo], ow, oh)
    if colorimetry:
        oi.set_colorimetry(matrix=colorimetry[0], range=colorimetry[1], chroma_site=colorimetry[2])
    el.set_info(ii, oi)
    assert int(el.plan_info().kernel_variant) == 5
    dst = torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda")
    el.transform_frame(torch.from_numpy(frame).cuda(), dst)
    torch.cuda.synchronize()
    return [dst.cpu().numpy()], oi


def expected(size, method, frame, fi, fo, colorimetry=None):
    d = ob.vcs_desc(*size, method, in_fmt=ob.FMT[fi], out_fmt=ob.FMT[fo])
    if colorimetry:
        d.out_matrix, d.out_range, d.out_chroma_site = colorimetry
    return ob.oracle_vcs_convert(d, frame)


# large shapes: NV12 output, bilinear / lanczos only (the CPU oracle needs seconds per frame there)
RGB420_CASES = [(fo, s, m) for fo in YUV_OUT for s in SIZES for m in (0, 1, 3, 4, 9)
                if not (s[0] * s[1] > 500_000 and (fo != "NV12" or m not in (1, 3)))]


@pytest.mark.parametrize("fo,size,method", RGB420_CASES, ids=lambda v: "-".join(str(x) for x in v) if isinstance(v, tuple) else str(v))
def test_rgb_to_420_matches_oracle(cuda_device, fo, size, method):
    from test_vcs_cross_gpu import planes_equal
    iw, ih, ow, oh = size
    big = iw * ih > 500_000
    for fi in (["BGRA"] if big else RGB_IN):
        frame = rgb_frame(iw, ih, 5)
        want = expected(size, method, frame, fi, fo)
        (got,), oi = convert(size, method, frame, fi, fo)
        bad = planes_equal(got, want, oi, ow, oh, fo in ("NV12", "NV21"))
        assert not bad, f"{fi}: {bad}"


@pytest.mark.parametrize("colorimetry", [(3, 2, 2), (4, 1, 1), (6, 2, 6), (2, 1, 4), (5, 2, 1)])
def test_rgb_to_420_colorimetry(cuda_device, colorimetry):
    from test_vcs_cross_gpu import planes_equal
    for size in [(64, 48, 40, 30), (40, 30, 64, 48), (33, 33, 33, 33)]:
        frame = rgb_frame(size[0], size[1], 7)
        want = expected(size, 3, frame, "BGRA", "NV12", colorimetry)
        (got,), oi = convert(size, 3, frame, "BGRA", "NV12", colorimetry)
        assert not planes_equal(got, want, oi, size[2], size[3], True)


@pytest.mark.parametrize("method", [0, 1, 3, 4, 9], ids=["nearest", "bilinear", "lanczos", "bilinear2", "mitchell"])
@pytest.mark.parametrize("size", [(64, 48, 32, 24), (40, 30, 64, 48), (65, 49, 33, 26), (33, 17, 20, 31), (100, 100, 150, 50),
                                  (40, 90, 40, 31), (64, 48, 64, 24), (64, 48, 32, 48), (3, 5, 7, 2), (1, 1, 4, 4),
                                  (50, 21, 50, 21), (1920, 1080, 640, 360), (640, 360, 1280, 720), (1918, 1080, 1279, 721),
                                  (402, 300, 150, 100)], ids=lambda s: "%dx%d-%dx%d" % s)
def test_rgb_same_format_scaling_matches_oracle(cuda_device, size, method):
    """a compositor's scaled RGBA pads: one plane of 4-byte pixels through vcs_planes_fast_kernel (NC = 4; the byte order
    change is one PRMT at the store) or, for shapes it declines, the byte-wise vcs_planes_kernel (ne = 4)"""
    import torch
    import gstreamer_b200 as g
    iw, ih, ow, oh = size
    pairs = [("BGRA", "BGRA"), ("xRGB", "BGRA")] if iw * ih > 500_000 else [("BGRA", "BGRA"), ("RGBA", "RGBA"), ("ARGB", "ARGB"), ("xBGR", "xBGR"),
                                                            ("BGRA", "RGBA"), ("ARGB", "BGRx"), ("RGBx", "ABGR"), ("xRGB", "BGRA")]
    for fmt, fmt_out in pairs:                      # same format: one-plane rows; another byte order: matrix-free chain
        frame = rgb_frame(iw, ih, 11)
        want = ob.oracle_vcs_convert(ob.vcs_desc(iw, ih, ow, oh, method, in_fmt=ob.FMT[fmt], out_fmt=ob.FMT[fmt_out]), frame)
        el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
        ii, oi = g.VideoInfo(ob.FMT[fmt], iw, ih), g.VideoInfo(ob.FMT[fmt_out], ow, oh)
        el.set_info(ii, oi)
        assert int(el.plan_info().kernel_variant) == 4
        dst = torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda")
        el.transform_frame(torch.from_numpy(frame).cuda(), dst)
        torch.cuda.synchronize()
        got = dst.cpu().numpy()
        bad = np.argwhere(got != want)
        assert bad.size == 0, f"{fmt}->{fmt_out}: {len(bad)} bytes differ, first at {bad[:4].ravel().tolist()}"


@pytest.mark.parametrize("fi", ["YUY2", "UYVY", "YVYU", "Y42B", "Y444"])
@pytest.mark.parametrize("size", [(64, 48, 32, 24), (64, 48, 96, 72), (65, 49, 33, 26), (33, 17, 20, 31), (50, 21, 50, 21),
                                  (100, 100, 150, 50), (40, 90, 40, 31), (1, 1, 5, 4), (1920, 1080, 1280, 720)],
                         ids=lambda s: "%dx%d-%dx%d" % s)
def test_422_444_inputs_match_oracle(cuda_device, fi, size):
    """capture formats -> packed RGB through the generic kernel"""
    import torch
    import gstreamer_b200 as g
    iw, ih, ow, oh = size
    for method in ([1] if iw * ih > 500_000 else [0, 1, 3, 9]):
        for site in (1, 2):
            d = ob.vcs_desc(iw, ih, ow, oh, method, in_fmt=ob.FMT[fi], out_fmt=ob.FMT["BGRA"], site=site)
            frame = np.random.default_rng(method).integers(0, 256, ob.vcs_sizes(d)[0], dtype=np.uint8)
            want = ob.oracle_vcs_convert(d, frame)
            el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
            ii, oi = g.VideoInfo(ob.FMT[fi], iw, ih), g.VideoInfo(ob.FMT["BGRA"], ow, oh)
            ii.set_colorimetry(chroma_site=site)
            el.set_info(ii, oi)
            dst = torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda")
            el.transform_frame(torch.from_numpy(frame).cuda(), dst)
            torch.cuda.synchronize()
            got = dst.cpu().numpy()
            bad = np.argwhere(got != want)
            assert bad.size == 0, f"m{method} site{site}: {len(bad)} bytes differ, first at {bad[:4].ravel().tolist()}"


@pytest.mark.parametrize("pair", [("YUY2", "I420"), ("UYVY", "YV12"), ("UYVY", "I420"), ("YUY2", "YV12"), ("YVYU", "I420"), ("YUY2", "NV12"),
                                  ("UYVY", "NV21"), ("YVYU", "NV12")], ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("size", [(64, 48, 64, 48), (50, 21, 50, 21), (33, 17, 33, 17), (1, 1, 1, 1), (2, 3, 2, 3), (1282, 722, 1282, 722),
                                  (1920, 1080, 1920, 1080), (64, 48, 32, 24), (64, 48, 96, 72), (33, 17, 20, 31), (100, 100, 150, 50),
                                  (1920, 1080, 1280, 720)], ids=lambda s: "%dx%d-%dx%d" % s)
def test_packed_422_to_420_matches_oracle(cuda_device, pair, size):
    """capture -> encoder: the table rows YUY2 / UYVY -> I420 / YV12 at an unchanged size (vcs_yuy2_420_kernel), the chain
    (vcs_yuy2_ayuv_kernel -> word-wide scaler -> vcs_rgb420_kernel<MATRIX = false>) for every other pair or size"""
    import torch
    import gstreamer_b200 as g
    from gstreamer_b200.video import transfer_colorimetry_from_input
    from test_vcs_cross_gpu import planes_equal
    fi, fo = pair
    iw, ih, ow, oh = size
    table_row = fi in ("YUY2", "UYVY") and fo in ("I420", "YV12") and (iw, ih) == (ow, oh)
    for method in ([1] if iw * ih > 500_000 else [0, 1, 3, 9]):
        for site in (1, 2):
            d = ob.vcs_desc(iw, ih, ow, oh, method, in_fmt=ob.FMT[fi], out_fmt=ob.FMT[fo], site=site)
            frame = np.random.default_rng(method + 7).integers(0, 256, ob.vcs_sizes(d)[0], dtype=np.uint8)
            want = ob.oracle_vcs_convert(d, frame)
            el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
            ii, oi = g.VideoInfo(ob.FMT[fi], iw, ih), g.VideoInfo(ob.FMT[fo], ow, oh)
            ii.set_colorimetry(chroma_site=site)
            transfer_colorimetry_from_input(ii, oi)
            el.set_info(ii, oi)
            # the chain: unpack + chroma up-sampling kernel, word-wide scaler, down-sample + pack kernel - or, for shapes
            # the scaler declines, the generic kernel
            assert el.kernel_name() in (("vcs_yuy2_420_kernel",) if table_row else ("vcs_yuy2_ayuv_kernel", "vcs_generic_kernel")), el.kernel_name()
            dst = torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda")
            el.transform_frame(torch.from_numpy(frame).cuda(), dst)
            torch.cuda.synchronize()
            got = dst.cpu().numpy()
            if table_row and (ow & 1):
                # the reference's convert_YUY2_I420 copies the luma in whole pixel pairs: on a line pair an odd width writes one
                # byte of row padding (the oracle, pinned against it, does too) - checked here, then hidden from planes_equal
                idx = int(oi.c.offset[0]) + np.arange(oh & ~1) * int(oi.c.stride[0]) + ow
                assert np.array_equal(got[idx], want[idx]), "padding byte of the pair copy"
                got[idx] = 0x5A
            bad = planes_equal(got, want, oi, ow, oh, fo in ("NV12", "NV21"))
            assert not bad, f"m{method} site{site}: " + "; ".join(bad)


@pytest.mark.parametrize("pair", [("Y42B", "I420"), ("Y444", "YV12"), ("Y42B", "YV12"), ("Y444", "I420"), ("Y42B", "NV12"), ("Y444", "NV21")],
                         ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("size", [(64, 48, 64, 48), (50, 21, 50, 21), (33, 17, 33, 17), (2, 3, 2, 3), (64, 48, 32, 24), (64, 48, 96, 72),
                                  (33, 17, 20, 31), (100, 100, 150, 50), (64, 48, 64, 24), (64, 48, 128, 96), (1920, 1080, 1920, 1080),
                                  (1920, 1080, 1280, 720)], ids=lambda s: "%dx%d-%dx%d" % s)
def test_planar_422_444_to_420_matches_oracle(cuda_device, pair, size):
    """Y42B / Y444 -> I420 / YV12: the reference's plane-scaling rows on the plane kernels (kernel_variant 4), chroma planes
    with the input format's own geometry; -> NV12 / NV21: the chain (kernel_variant 5: generic kernel + vcs_down420_kernel)"""
    import torch
    import gstreamer_b200 as g
    from gstreamer_b200.video import transfer_colorimetry_from_input
    from test_vcs_cross_gpu import planes_equal
    fi, fo = pair
    iw, ih, ow, oh = size
    for method in ([1, 3] if iw * ih > 500_000 else [0, 1, 3, 4, 9]):
        d = ob.vcs_desc(iw, ih, ow, oh, method, in_fmt=ob.FMT[fi], out_fmt=ob.FMT[fo])
        frame = np.random.default_rng(method + 3).integers(0, 256, ob.vcs_sizes(d)[0], dtype=np.uint8)
        want = ob.oracle_vcs_convert(d, frame)
        el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
        ii, oi = g.VideoInfo(ob.FMT[fi], iw, ih), g.VideoInfo(ob.FMT[fo], ow, oh)
        transfer_colorimetry_from_input(ii, oi)
        el.set_info(ii, oi)
        semi = fo in ("NV12", "NV21")
        assert int(el.plan_info().kernel_variant) == (5 if semi else 4)
        dst = torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda")
        el.transform_frame(torch.from_numpy(frame).cuda(), dst)
        torch.cuda.synchronize()
        bad = planes_equal(dst.cpu().numpy(), want, oi, ow, oh, semi)
        assert not bad, f"m{method}: " + "; ".join(bad)
