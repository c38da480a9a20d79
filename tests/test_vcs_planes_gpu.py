"""YUV -> same YUV family (NV12->NV12, NV21->NV21, I420/YV12 -> I420/YV12): the reference's plane-scaling fast path
(convert_scale_planes): luma with the element's method, chroma with the linear chroma resampler, exact 2:1 / 1:2
steps by the averaging / doubling kernels — the transcoding-ladder case."""
import numpy as np
import pytest

from oracle import bindings as ob

pytestmark = pytest.mark.gpu

SIZES = [(64, 48, 32, 24), (64, 48, 128, 96), (64, 48, 40, 30), (64, 48, 100, 70), (65, 49, 33, 25), (33, 17, 20, 9),
         (64, 48, 64, 24), (64, 48, 32, 48), (64, 48, 64, 96), (64, 48, 128, 48), (640, 480, 320, 240), (320, 240, 640, 480),
         (1920, 1080, 1280, 720), (100, 100, 50, 150), (3, 5, 7, 2), (2, 2, 1, 1), (1, 1, 2, 2), (16, 16, 16, 16),
         (3840, 2160, 1920, 1080), (1280, 720, 854, 480)]
PAIRS = [("NV12", "NV12"), ("NV21", "NV21"), ("I420", "I420"), ("YV12", "YV12"), ("I420", "YV12"), ("YV12", "I420")]


def _convert(iw, ih, ow, oh, method, frame, in_fmt, out_fmt):
    import torch
    import gstreamer_b200 as g
    el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
    ii, oi = g.VideoInfo(in_fmt, iw, ih), g.VideoInfo(out_fmt, ow, oh)
    el.set_info(ii, oi)
    assert int(el.plan_info().kernel_variant) == 4
    dst = torch.full((oi.size,), 0x5A, dtype=torch.uint8, device="cuda")
    el.transform_frame(torch.from_numpy(frame).cuda(), dst)
    torch.cuda.synchronize()
    return [dst.cpu().numpy()], oi


# large shapes: bilinear / lanczos on the same-format pairs only (the CPU oracle needs seconds per frame there)
PLANE_CASES = [(p, s, m) for p in PAIRS for s in SIZES for m in (0, 1, 3, 4, 9)
               if not (s[0] * s[1] > 2_000_000 and (p[0] != p[1] or m not in (1, 3)))]


@pytest.mark.parametrize("pair,size,method", PLANE_CASES, ids=lambda v: "-".join(str(x) for x in v) if isinstance(v, tuple) else str(v))
def test_plane_scaling_matches_oracle(cuda_device, pair, size, method):
    iw, ih, ow, oh = size
    fi, fo = ob.FMT[pair[0]], ob.FMT[pair[1]]
    frame = ob.i420_random_frame(iw, ih, 5) if pair[0] in ("I420", "YV12") else ob.nv12_random_frame(iw, ih, 5)
    d = ob.vcs_desc(iw, ih, ow, oh, method, in_fmt=fi, out_fmt=fo)
    want = ob.oracle_vcs_convert(d, frame)
    (got,), oi = _convert(iw, ih, ow, oh, method, frame, fi, fo)
    assert got.size == want.size
    # compare the pixel bytes of every plane (row padding is never written: it keeps the 0x5A fill)
    semi = pair[1] in ("NV12", "NV21")
    for p in range(2 if semi else 3):
        w = ow if p == 0 else ((ow + 1) // 2) * (2 if semi else 1)
        h = oh if p == 0 else (oh + 1) // 2
        st, off = oi.stride[p], oi.offset[p]
        g_pl = got[off: off + st * h].reshape(h, st)
        w_pl = want[off: off + st * h].reshape(h, st)
        bad = np.argwhere(g_pl[:, :w] != w_pl[:, :w])
        assert bad.size == 0, f"plane {p}: {len(bad)} bytes differ, first at {bad[:4].tolist()}"
        assert (g_pl[:, w:] == 0x5A).all()

