"""Planar RGB outputs (RGBP / BGRP) on the device, byte for byte against the oracle: every sink format, every fast
kernel's planar store form, the headline shapes, batches, the host path, borders and arbitrary plane layouts."""
import numpy as np
import pytest

from oracle import bindings as ob
from rgbp_oracle import FMT, oracle_rgbp

pytestmark = pytest.mark.gpu

YUV420 = ["NV12", "NV21", "I420", "YV12"]
RGB = ["BGRA", "RGBA", "ARGB", "ABGR", "BGRx", "RGBx", "xRGB", "xBGR"]
CAPTURE = ["YUY2", "UYVY", "YVYU", "Y42B", "Y444"]
OUTS = ["RGBP", "BGRP"]


def _frame(fmt, iw, ih, seed):
    d = ob.vcs_desc(iw, ih, iw, ih, 1, in_fmt=FMT[fmt], out_fmt=12)
    return np.random.default_rng(seed).integers(0, 256, ob.vcs_sizes(d)[0], dtype=np.uint8)


def _want(fi, fo, size, method, frame, site=None, layout=None, dest=None, border=0xff000000):
    return oracle_rgbp(fi, fo, size, method, frame, site=site, layout=layout, dest=dest, border=border)


def _element(fi, fo, size, method, site=None, layout=None, add_borders=False):
    import gstreamer_b200 as g
    iw, ih, ow, oh = size
    el = g.CudaVideoConvertScale(add_borders=add_borders, method=method, cuda_device_id=0)
    ii = g.VideoInfo(FMT[fi], iw, ih)
    if site is not None:
        ii.set_colorimetry(chroma_site=site)
    oi = g.VideoInfo(FMT[fo], ow, oh)
    if layout:
        oi.set_layout(*layout)
    el.set_info(ii, oi)
    return el, oi


def _run(el, oi, frame):
    import torch
    dst = torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda")
    el.transform_frame(torch.from_numpy(frame).cuda(), dst)
    torch.cuda.synchronize()
    return dst.cpu().numpy()


def _check(got, want, tag):
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{tag}: {bad.size} bytes differ, first at {bad[:8]}: got {got[bad[:8]]} want {want[bad[:8]]}"


def _odd_layout(ow, oh, order=(2, 0, 1)):
    strides = [ow + 5, ow + 3, ow + 9]
    offs, pos = [0, 0, 0], 3
    for k in order:
        offs[k] = pos
        pos += strides[k] * oh + 7
    return strides, offs


# (sink, size, method, site, kernel that must run)
KERNEL_CASES = [
    ("NV12", (512, 248, 256, 124), 3, 2, "vcs_lanczos2_v2_kernel"),
    ("NV21", (512, 248, 256, 124), 9, 2, "vcs_lanczos2_v2_kernel"),
    ("I420", (512, 248, 256, 124), 3, 2, "vcs_lanczos2_v2_kernel"),
    ("YV12", (512, 248, 256, 124), 7, 2, "vcs_lanczos2_v2_kernel"),
    ("NV12", (640, 360, 427, 240), 1, 2, "vcs_light_kernel"),
    ("NV21", (320, 180, 480, 90), 1, 1, "vcs_light_kernel"),          # vertical pass first
    ("I420", (98, 66, 98, 66), 1, 1, "vcs_light_kernel"),             # same size: the chain, not the I420 table row
    ("YV12", (640, 360, 427, 240), 1, 2, "vcs_light_kernel"),
    ("NV12", (648, 360, 427, 240), 3, 2, "vcs_ntap_kernel"),
    ("NV12", (200, 120, 300, 90), 9, 2, "vcs_ntap_kernel"),           # vertical pass first
    ("I420", (641, 481, 320, 200), 3, 1, "vcs_ntap_kernel"),
    ("NV21", (98, 66, 45, 37), 3, 1, "vcs_ntap_kernel"),
] + [(f, (98, 66, 45, 37), 3, 2, "vcs_generic_kernel") for f in CAPTURE] + \
    [(f, (98, 66, 45, 37), 3, None, "vcs_rgb_deinterleave_kernel") for f in RGB] + \
    [(f, (98, 66, 98, 66), 1, None, "vcs_rgb_deinterleave_kernel") for f in ("BGRA", "xBGR")]


@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("case", KERNEL_CASES, ids=lambda c: "%s-%dx%d-%dx%d-m%d" % (c[0], *c[1], c[2]))
def test_every_sink_and_kernel(cuda_device, case, fo):
    fi, size, method, site, kernel = case
    frame = _frame(fi, size[0], size[1], 3)
    el, oi = _element(fi, fo, size, method, site)
    assert el.kernel_name() == kernel
    _check(_run(el, oi, frame), _want(fi, fo, size, method, frame, site), f"{fi}->{fo} {kernel}")
    if fi not in RGB:
        el.set_kernel_variant(0)
        _check(_run(el, oi, frame), _want(fi, fo, size, method, frame, site), f"{fi}->{fo} generic")


@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("size,method,kernel", [((3840, 2160, 1920, 1080), 3, "vcs_lanczos2_v2_kernel"),
                                                ((3840, 2160, 1920, 1080), 1, "vcs_light_kernel"),
                                                ((1920, 1080, 1280, 720), 1, "vcs_light_kernel"),
                                                ((1920, 1080, 640, 640), 3, "vcs_ntap_kernel")],
                         ids=["4k-1080p-lanczos", "4k-1080p-bilinear", "1080p-720p-bilinear", "1080p-640-lanczos"])
def test_headline_shapes(cuda_device, size, method, kernel, fo):
    frame = ob.nv12_random_frame(size[0], size[1], 99)
    el, oi = _element("NV12", fo, size, method)
    assert el.kernel_name() == kernel
    _check(_run(el, oi, frame), _want("NV12", fo, size, method, frame), kernel)


def test_default_layout_is_a_chw_tensor(cuda_device):
    import torch
    frame = ob.nv12_random_frame(3840, 2160, 7)
    el, oi = _element("NV12", "RGBP", (3840, 2160, 1920, 1080), 3)
    chw = torch.empty((3, 1080, 1920), dtype=torch.uint8, device="cuda")
    assert oi.size == chw.numel()
    el.transform_frame(torch.from_numpy(frame).cuda(), chw)
    torch.cuda.synchronize()
    want = _want("NV12", "RGBP", (3840, 2160, 1920, 1080), 3, frame).reshape(3, 1080, 1920)
    assert torch.equal(chw.cpu(), torch.from_numpy(want))


@pytest.mark.parametrize("fi,fo,method", [("NV12", "RGBP", 3), ("I420", "BGRP", 1), ("BGRA", "RGBP", 3), ("YUY2", "BGRP", 9)])
def test_batch_of_64(cuda_device, fi, fo, method):
    import torch
    size = (256, 144, 128, 72) if method == 3 else (256, 144, 170, 96)
    el, oi = _element(fi, fo, size, method, site=2 if fi not in RGB else None)
    frames = [_frame(fi, size[0], size[1], 100 + i) for i in range(64)]
    src = [torch.from_numpy(f).cuda() for f in frames]
    dst = [torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda") for _ in frames]
    el.transform_frames(src, dst)
    torch.cuda.synchronize()
    for i in (0, 1, 31, 63):
        _check(dst[i].cpu().numpy(), _want(fi, fo, size, method, frames[i], 2 if fi not in RGB else None), f"frame {i}")


@pytest.mark.parametrize("fi,fo", [("NV12", "RGBP"), ("BGRA", "BGRP")])
def test_host_frames_pinned(cuda_device, fi, fo):
    import gstreamer_b200 as g
    size = (640, 360, 320, 180)
    el, oi = _element(fi, fo, size, 3)
    ins, outs, keep = [], [], []
    n = 40
    frames = [_frame(fi, 640, 360, 200 + i) for i in range(n)]
    for f in frames:
        hi, ho = g.PinnedBuffer(f.size), g.PinnedBuffer(oi.size)
        hi.array[:] = f
        ins.append(hi)
        outs.append(ho)
    el.transform_host_frames([b.ptr for b in ins], [b.ptr for b in outs])
    for i in (0, 17, n - 1):
        _check(outs[i].array.copy(), _want(fi, fo, size, 3, frames[i]), f"host frame {i}")


@pytest.mark.parametrize("fi", ["NV12", "I420", "BGRA", "YUY2"])
@pytest.mark.parametrize("fo", OUTS)
def test_add_borders(cuda_device, fi, fo):
    size = (640, 480, 640, 360)                      # 4:3 into 16:9: pillar boxes
    frame = _frame(fi, 640, 480, 1)
    el, oi = _element(fi, fo, size, 3, add_borders=True)
    dest = ob.vcs_borders(*size)
    assert dest != (0, 0, 640, 360)
    _check(_run(el, oi, frame), _want(fi, fo, size, 3, frame, dest=dest), f"{fi}->{fo} borders {dest}")


@pytest.mark.parametrize("fo", OUTS)
@pytest.mark.parametrize("fi,size,method,kernel", [("NV12", (512, 248, 256, 124), 3, "vcs_lanczos2_v2_kernel"),
                                                   ("NV12", (640, 360, 427, 240), 1, "vcs_light_kernel"),
                                                   ("I420", (648, 360, 427, 240), 3, "vcs_ntap_kernel"),
                                                   ("Y444", (98, 66, 45, 37), 3, "vcs_generic_kernel"),
                                                   ("RGBA", (98, 66, 45, 37), 3, "vcs_rgb_deinterleave_kernel")])
def test_strides_above_width_unaligned_offsets_padding_untouched(cuda_device, fi, fo, size, method, kernel):
    ow, oh = size[2], size[3]
    layout = _odd_layout(ow, oh)
    frame = _frame(fi, size[0], size[1], 4)
    el, oi = _element(fi, fo, size, method, site=2 if fi not in RGB else None, layout=layout)
    assert el.kernel_name() == kernel
    got = _run(el, oi, frame)
    _check(got, _want(fi, fo, size, method, frame, site=2 if fi not in RGB else None, layout=layout), kernel)
    for k in range(3):                             # bytes between width and stride, and between planes, keep 0x5A
        rows = got[layout[1][k]: layout[1][k] + layout[0][k] * oh].reshape(oh, layout[0][k])
        assert (rows[:, ow:] == 0x5A).all()
    assert (got[:3] == 0x5A).all()
