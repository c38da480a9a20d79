"""vcs_l2mma_kernel (kernel_variant 6): the 2:1 / 8-tap kernel with both FIR passes on the integer tensor path
(mma.sync.m16n8k32 u8 x s8).  Bit-exact under emulation (tests/test_emu_kernels.py) and on the device; slower than the SIMT kernel
(DESIGN.md), so it stays an opt-in variant."""
import os

import numpy as np
import pytest

from oracle import bindings as ob

pytestmark = [pytest.mark.gpu]

SIZES = [(16, 16), (64, 48), (256, 144), (496, 272), (1920, 1088), (3840, 2160)]   # output sizes must be multiples of 8
METHODS = [3, 5, 6, 7, 8, 9]


def convert(iw, ih, method, frames, in_fmt=23, out_fmt=12, matrix=None, rng=None):
    """one frame, or a batch (a list of frames) in one transform_frames call"""
    import torch
    import gstreamer_b200 as g
    el = g.CudaVideoConvertScale(add_borders=False, method=method)
    ii = g.VideoInfo(in_fmt, iw, ih).set_colorimetry(chroma_site=2, matrix=matrix, range=rng)
    oi = g.VideoInfo(out_fmt, iw // 2, ih // 2)
    el.set_info(ii, oi)
    el.set_kernel_variant(6)
    assert el.plan_info().kernel_variant == 6
    src = [torch.from_numpy(f).cuda() for f in (frames if isinstance(frames, list) else [frames])]
    dst = [torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda") for _ in src]
    if len(src) == 1:
        el.transform_frame(src[0], dst[0])
    else:
        el.transform_frames(src, dst)
    torch.cuda.synchronize()
    return [d.cpu().numpy() for d in dst]


MMA_CASES = [(s, m) for m in METHODS for s in SIZES if m == 3 or s[0] <= 2000]      # full size: the headline method only


@pytest.mark.parametrize("size,method", MMA_CASES, ids=lambda v: "%dx%d" % v if isinstance(v, tuple) else str(v))
def test_tensor_path_matches_oracle(cuda_device, size, method):
    iw, ih = size
    frame = ob.nv12_random_frame(iw, ih, seed=iw + method)
    want = ob.oracle_vcs_convert(ob.vcs_desc(iw, ih, iw // 2, ih // 2, method, site=2), frame)
    (got,) = convert(iw, ih, method, frame)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[:6].tolist()}: got {got[bad[:6]]} want {want[bad[:6]]}"


@pytest.mark.parametrize("in_fmt", ["NV12", "NV21"])
@pytest.mark.parametrize("out_fmt", ["BGRA", "RGBA", "ARGB", "ABGR", "xRGB"])
def test_tensor_path_formats_and_batch(cuda_device, in_fmt, out_fmt):
    iw, ih = 496, 272
    d = ob.vcs_desc(iw, ih, iw // 2, ih // 2, 3, in_fmt=ob.FMT[in_fmt], out_fmt=ob.FMT[out_fmt], site=2, matrix=4, rng=1)
    frames = [ob.nv12_random_frame(iw, ih, seed=3 + k) for k in range(3)]          # a frame of its own in every slot
    for k, got in enumerate(convert(iw, ih, 3, frames, ob.FMT[in_fmt], ob.FMT[out_fmt], matrix=4, rng=1)):
        assert np.array_equal(got, ob.oracle_vcs_convert(d, frames[k])), f"frame {k}"
