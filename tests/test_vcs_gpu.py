"""Parity of the CUDA convert+scale path (through the C-ABI) against the CPU oracle.

Bit-exactness is the bar: every output byte must equal the oracle's, which is itself
pinned to the reference's own sources (tests/test_oracle_vs_ref.py).
"""
import numpy as np
import pytest

from oracle import bindings as ob

pytestmark = pytest.mark.gpu

# size matrix after the reference's own element test
# (gst-plugins-base/tests/check/elements/videoscale.c:451-492) plus the BASELINE configs
SIZES = [
    (640, 480, 320, 240), (320, 240, 640, 480), (320, 240, 320, 240),
    (641, 481, 111, 30), (111, 30, 641, 481),
    (641, 481, 30, 111), (30, 111, 641, 481),
    (1, 1, 1, 1), (2, 2, 1, 1), (1, 1, 2, 2), (16, 16, 16, 16), (3, 5, 7, 2), (17, 33, 64, 7),
    (100, 100, 150, 50), (100, 100, 50, 150), (720, 480, 640, 360), (641, 481, 640, 480),
]
METHODS = list(range(10))


def _run_gpu(iw, ih, ow, oh, method, frame, in_fmt=23, out_fmt=12, site=None, matrix=None, rng=None):
    import torch
    import gstreamer_b200 as g
    el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
    ii = g.VideoInfo(in_fmt, iw, ih)
    ii.set_colorimetry(matrix=matrix, range=rng, chroma_site=site)
    oi = g.VideoInfo(out_fmt, ow, oh)
    el.set_info(ii, oi)
    assert ii.size == frame.size
    dst = torch.full((oi.size,), 0xA5, dtype=torch.uint8, device="cuda")
    el.transform_frame(torch.from_numpy(frame).cuda(), dst)
    torch.cuda.synchronize()
    return [dst.cpu().numpy()]


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d-%dx%d" % s)
@pytest.mark.parametrize("method", METHODS)
def test_matches_oracle(cuda_device, size, method):
    iw, ih, ow, oh = size
    d = ob.vcs_desc(iw, ih, ow, oh, method)
    frame = ob.nv12_random_frame(iw, ih, seed=iw * 7 + oh)
    want = ob.oracle_vcs_convert(d, frame)
    got = _run_gpu(iw, ih, ow, oh, method, frame)[0]
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[:8]}: got {got[bad[:8]]} want {want[bad[:8]]}"


@pytest.mark.parametrize("out_fmt", ["RGBx", "BGRx", "xRGB", "xBGR", "RGBA", "BGRA", "ARGB", "ABGR"])
@pytest.mark.parametrize("in_fmt", ["NV12", "NV21"])
def test_formats(cuda_device, in_fmt, out_fmt):
    iw, ih, ow, oh = 98, 66, 45, 37
    d = ob.vcs_desc(iw, ih, ow, oh, 3, in_fmt=ob.FMT[in_fmt], out_fmt=ob.FMT[out_fmt])
    frame = ob.nv12_random_frame(iw, ih, seed=5)
    want = ob.oracle_vcs_convert(d, frame)
    got = _run_gpu(iw, ih, ow, oh, 3, frame, in_fmt=ob.FMT[in_fmt], out_fmt=ob.FMT[out_fmt])[0]
    assert np.array_equal(got, want)


@pytest.mark.parametrize("site", [1, 2, 4, 6])
@pytest.mark.parametrize("matrix,rng", [(3, 2), (4, 2), (4, 1), (6, 2), (2, 1), (5, 2)])
def test_colorimetry_and_siting(cuda_device, site, matrix, rng):
    iw, ih, ow, oh = 130, 74, 65, 37
    d = ob.vcs_desc(iw, ih, ow, oh, 3, site=site, matrix=matrix, rng=rng)
    frame = ob.nv12_random_frame(iw, ih, seed=site * 10 + matrix)
    want = ob.oracle_vcs_convert(d, frame)
    got = _run_gpu(iw, ih, ow, oh, 3, frame, site=site, matrix=matrix, rng=rng)[0]
    assert np.array_equal(got, want)


@pytest.mark.parametrize("cfg", [(1920, 1080, 1280, 720, 1), (3840, 2160, 1920, 1080, 3)],
                         ids=["C1-1080p-bilinear-720p", "C2-4K-lanczos-1080p"])
@pytest.mark.parametrize("content", ["random", "smpte"])
def test_baseline_configs_full_size(cuda_device, cfg, content):
    iw, ih, ow, oh, method = cfg
    d = ob.vcs_desc(iw, ih, ow, oh, method)
    frame = ob.nv12_random_frame(iw, ih, 3) if content == "random" else ob.nv12_smpte_like_frame(iw, ih, 3)
    want = ob.oracle_vcs_convert(d, frame)
    got = _run_gpu(iw, ih, ow, oh, method, frame)[0]
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[:8]}"


def test_custom_strides_and_offsets(cuda_device):
    """GstCudaMemory hands out one pitched allocation with a common pitch for all planes
    (gst-plugins-bad/gst-libs/gst/cuda/gstcudamemory.cpp:194-345): honour arbitrary layouts."""
    import torch
    import gstreamer_b200 as g
    iw, ih, ow, oh = 250, 140, 125, 70
    d = ob.vcs_desc(iw, ih, ow, oh, 3)
    frame = ob.nv12_random_frame(iw, ih, 2)
    want = ob.oracle_vcs_convert(d, frame).reshape(oh, ow * 4)
    st = (iw + 3) & ~3
    pitch, opitch = 512, 1024
    padded = np.full(pitch * (ih + ih // 2) + 256, 0x33, dtype=np.uint8)
    y = frame[: st * ih].reshape(ih, st)
    uv = frame[st * ih:].reshape(ih // 2, st)
    padded[256: 256 + pitch * ih].reshape(ih, pitch)[:, :st] = y
    padded[256 + pitch * ih:].reshape(ih // 2, pitch)[:, :st] = uv
    ii = g.VideoInfo(23, iw, ih).set_layout([pitch, pitch], [256, 256 + pitch * ih])
    oi = g.VideoInfo(12, ow, oh).set_layout([opitch], [64])
    el = g.CudaVideoConvertScale(add_borders=False, method=3)
    el.set_info(ii, oi)
    src = torch.from_numpy(padded).cuda()
    dst = torch.full((64 + opitch * oh,), 0x5A, dtype=torch.uint8, device="cuda")
    el.transform_frame(src, dst)
    torch.cuda.synchronize()
    out = dst.cpu().numpy()
    assert (out[:64] == 0x5A).all()
    rows = out[64:].reshape(oh, opitch)
    assert np.array_equal(rows[:, : ow * 4], want)
    assert (rows[:, ow * 4:] == 0x5A).all()          # padding untouched


def test_host_path_round_trip(cuda_device):
    """system-memory peers: pinned staging H2D -> kernel -> D2H inside the library"""
    import gstreamer_b200 as g
    iw, ih, ow, oh = 640, 360, 320, 180
    d = ob.vcs_desc(iw, ih, ow, oh, 3)
    el = g.CudaVideoConvertScale(add_borders=False, method=3)
    ii, oi = g.VideoInfo(23, iw, ih), g.VideoInfo(12, ow, oh)
    el.set_info(ii, oi)
    n = 9
    ins = [g.PinnedBuffer(ii.size) for _ in range(n)]
    outs = [g.PinnedBuffer(oi.size) for _ in range(n)]
    wants = []
    for k, b in enumerate(ins):
        f = ob.nv12_random_frame(iw, ih, 100 + k)
        b.array[:] = f
        wants.append(ob.oracle_vcs_convert(d, f))
    el.transform_host_frames([b.ptr for b in ins], [b.ptr for b in outs])
    for k in range(n):
        assert np.array_equal(outs[k].array, wants[k]), f"frame {k}"


def test_properties_full_size(cuda_device):
    """size-independent checks at BASELINE size: away from the frame edges (where the
    reference's folded 6-bit taps need not sum to 64) a flat frame stays flat and alpha is
    opaque everywhere; a frame and its batch-mates produce identical bytes"""
    iw, ih, ow, oh = 3840, 2160, 1920, 1080
    st = iw
    frame = np.empty(st * ih * 3 // 2, dtype=np.uint8)
    frame[: st * ih] = 126
    frame[st * ih:] = 128
    got = _run_gpu(iw, ih, ow, oh, 3, frame)[0].reshape(oh, ow, 4)
    inner = got[4:-4, 4:-4]
    assert (inner == inner[0, 0]).all()
    assert (got[..., 3] == 255).all()
    assert tuple(inner[0, 0]) == (126, 126, 126, 255)       # Y=126,U=V=128 -> grey 126 via p1=298


def test_linearity_of_luma_steps_full_size(cuda_device):
    """exact property at BASELINE size: adding a constant to a flat-chroma luma plane far from
    saturation shifts every interior output by round-trip of the same matrix (checked against
    the oracle on a 64-row strip of the same frame, which shares all horizontal taps)"""
    iw, ih, ow, oh = 3840, 2160, 1920, 1080
    frame = ob.nv12_smpte_like_frame(iw, ih, 9)
    got = _run_gpu(iw, ih, ow, oh, 3, frame)[0].reshape(oh, ow, 4)
    # rows 8..23 of the output only depend on input rows 13..50; crop a strip and re-run the
    # oracle on it: interior rows must agree byte for byte
    strip_h = 128
    st = iw
    strip = np.concatenate([frame[: st * strip_h], frame[st * ih: st * ih + st * strip_h // 2]])
    d = ob.vcs_desc(iw, strip_h, ow, strip_h // 2, 3, site=2, matrix=3, rng=2)
    want = ob.oracle_vcs_convert(d, strip).reshape(strip_h // 2, ow, 4)
    assert np.array_equal(got[4:56], want[4:56])


@pytest.mark.parametrize("variant", [0, 2, 3])
def test_two_handles_share_a_kernel(cuda_device, variant):
    """The dynamic shared-memory limit is an attribute of the kernel FUNCTION: a second handle with a smaller footprint
    must not lower it under the first one (two converters in one process, a compositor's per-pad converters)."""
    import torch
    import gstreamer_b200 as g
    method = 1 if variant == 2 else 3
    big, small = (1920, 1080, 1280, 720), (64, 48, 32, 24)

    def make(size):
        el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
        ii, oi = g.VideoInfo(23, size[0], size[1]), g.VideoInfo(12, size[2], size[3])
        el.set_info(ii, oi)
        el.set_kernel_variant(variant)
        return el, ii, oi

    a, ii, oi = make(big)
    b, _, _ = make(small)          # created after, smaller tiles: used to shrink the shared attribute
    frame = ob.nv12_random_frame(big[0], big[1], seed=11)
    want = ob.oracle_vcs_convert(ob.vcs_desc(*big, method), frame)
    dst = torch.full((oi.size,), 0xA5, dtype=torch.uint8, device="cuda")
    a.transform_frame(torch.from_numpy(frame).cuda(), dst)
    torch.cuda.synchronize()
    assert np.array_equal(dst.cpu().numpy(), want)
