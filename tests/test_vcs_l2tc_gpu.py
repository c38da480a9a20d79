"""vcs_l2tc_kernel (kernel_variant 7): the exact-2:1 / 8-tap conversion with BOTH FIR passes on the Hopper tensor
cores (wgmma.mma_async s8 x u8, accumulators in registers, see gstreamer_b200/csrc/vcs_l2tc.cuh).  Bit-exact against
the oracle on every shape class the tiling distinguishes: partial strips (width not a multiple of 128 output columns),
partial row tiles (height not a multiple of 28 output rows), single-tile frames, frame-edge taps on all four sides,
both chroma orders, every 8-tap method, batches."""
import numpy as np
import pytest

from oracle import bindings as ob

pytestmark = [pytest.mark.gpu]

# input sizes: width % 16 == 0 (16-byte luma staging), height % 8 == 0 (output rows in groups of 4)
SIZES = [(32, 16), (256, 56), (272, 64), (512, 240), (1024, 448), (1936, 1096), (3840, 2160)]
METHODS = [3, 5, 6, 7, 8, 9]


def convert(iw, ih, method, frames, in_fmt=23, out_fmt=12, matrix=None, rng=None):
    """one frame, or a batch (a list of frames) in one transform_frames call"""
    import torch
    import gstreamer_b200 as g
    el = g.CudaVideoConvertScale(add_borders=False, method=method)
    ii = g.VideoInfo(in_fmt, iw, ih).set_colorimetry(chroma_site=2, matrix=matrix, range=rng)
    oi = g.VideoInfo(out_fmt, iw // 2, ih // 2)
    el.set_info(ii, oi)
    el.set_kernel_variant(7)
    assert el.plan_info().kernel_variant == 7
    src = [torch.from_numpy(f).cuda() for f in (frames if isinstance(frames, list) else [frames])]
    dst = [torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda") for _ in src]
    if len(src) == 1:
        el.transform_frame(src[0], dst[0])
    else:
        el.transform_frames(src, dst)
    torch.cuda.synchronize()
    return [d.cpu().numpy() for d in dst]


TC_CASES = [(s, m) for m in METHODS for s in SIZES if not (s[0] * s[1] > 2_000_000 and m not in (3, 9))]   # large: lanczos, mitchell


@pytest.mark.parametrize("size,method", TC_CASES, ids=lambda v: "%dx%d" % v if isinstance(v, tuple) else str(v))
def test_matches_oracle(cuda_device, size, method):
    iw, ih = size
    frame = ob.nv12_random_frame(iw, ih, seed=iw + method)
    want = ob.oracle_vcs_convert(ob.vcs_desc(iw, ih, iw // 2, ih // 2, method, site=2), frame)
    got = convert(iw, ih, method, frame)[0]
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[:8]}: got {got[bad[:8]]} want {want[bad[:8]]}"


@pytest.mark.parametrize("in_fmt,out_fmt", [("NV21", "BGRA"), ("NV12", "RGBA"), ("NV21", "xRGB"), ("NV12", "ABGR")])
def test_formats_and_batches(cuda_device, in_fmt, out_fmt):
    iw, ih = 528, 136
    frames = [ob.nv12_random_frame(iw, ih, seed=3 + k) for k in range(5)]          # a frame of its own in every slot
    d = ob.vcs_desc(iw, ih, iw // 2, ih // 2, 3, in_fmt=ob.FMT[in_fmt], out_fmt=ob.FMT[out_fmt], site=2)
    for k, got in enumerate(convert(iw, ih, 3, frames, in_fmt=ob.FMT[in_fmt], out_fmt=ob.FMT[out_fmt])):
        assert np.array_equal(got, ob.oracle_vcs_convert(d, frames[k])), f"frame {k}"


@pytest.mark.parametrize("matrix,rng", [(3, 2), (4, 1), (6, 2)])
def test_colorimetry(cuda_device, matrix, rng):
    iw, ih = 288, 120
    frame = ob.nv12_random_frame(iw, ih, seed=matrix)
    want = ob.oracle_vcs_convert(ob.vcs_desc(iw, ih, iw // 2, ih // 2, 3, site=2, matrix=matrix, rng=rng), frame)
    assert np.array_equal(convert(iw, ih, 3, frame, matrix=matrix, rng=rng)[0], want)


def test_extreme_pixels_saturate_like_the_reference(cuda_device):
    """all-0 / all-255 / checker inputs drive the negative lobes into both saturation ends"""
    iw, ih = 256, 64
    for fill in (0, 255, None):
        frame = np.full(iw * ih * 3 // 2, fill if fill is not None else 0, dtype=np.uint8)
        if fill is None:
            frame[::2] = 255
        want = ob.oracle_vcs_convert(ob.vcs_desc(iw, ih, iw // 2, ih // 2, 3, site=2), frame)
        assert np.array_equal(convert(iw, ih, 3, frame)[0], want)
