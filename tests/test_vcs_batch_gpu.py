"""The converter's batch dimension on the device: every row of tests/vcs_batch_cases.py on batches of distinct frames
(in separate allocations, and at shuffled offsets of one allocation), up to B200_VCS_MAX_BATCH frames on one handle,
against the oracle; then the headline workload exactly as bench.py runs it - 32 distinct 4K NV12 frames per
transform_frames call on a side stream - and 64 pinned frames through transform_host_frames."""
import hashlib

import numpy as np
import pytest

import vcs_batch_cases as vb
from oracle import bindings as ob

pytestmark = pytest.mark.gpu


class DevMem:
    """device buffers (torch's allocator: every buffer starts on a 512-byte boundary), on the default stream"""
    stream = None

    def buffer(self, nbytes):
        import torch
        return torch.full((nbytes,), vb.FILL, dtype=torch.uint8, device="cuda")

    def ptr(self, b):
        return b.data_ptr()

    def put(self, b, off, data):
        import torch
        b[off: off + data.size].copy_(torch.from_numpy(np.ascontiguousarray(data)))

    def get(self, b):
        return b.cpu().numpy()

    def sync(self):
        import torch
        torch.cuda.synchronize()


@pytest.mark.parametrize("row", vb.ROWS, ids=lambda r: r.id)
def test_batch_row(cuda_device, row, monkeypatch):
    """one handle: batches of 2, 5, 2, 64 and 3 distinct frames (the scratch image grows, its slices are reused), frames
    at shuffled offsets of one allocation with guards, one input twice, and a refused 65-frame batch"""
    from gstreamer_b200 import _lib
    mem = DevMem()
    h = vb.Handle(_lib.lib, row, monkeypatch)
    try:
        vb.check_batches(h, mem, (2, 5, 2, vb.MAX_BATCH, 3), seed=11)
        vb.check_unordered(h, mem, 5, seed=21)
        vb.check_aliased_input(h, mem, seed=31)
        vb.check_too_many(h, mem, seed=41)
    finally:
        h.close()


# ---- the headline workload ------------------------------------------------------------------------------------------
IW, IH, OW, OH = 3840, 2160, 1920, 1080
FRAMES = 32


@pytest.fixture(scope="module")
def headline(cuda_device):
    """bench.py's converter and frames: four random bases, frame k = base k % 4 with every 4099th byte raised by k"""
    import torch
    import gstreamer_b200 as g
    el = g.CudaVideoConvertScale(method=3, cuda_device_id=0)
    ii, oi = g.VideoInfo(g.VideoFormat.NV12, IW, IH), g.VideoInfo(g.VideoFormat.BGRA, OW, OH)
    el.set_info(ii, oi)
    assert el.kernel_name() == "vcs_lanczos2_v2_kernel"
    base = [torch.from_numpy(ob.nv12_random_frame(IW, IH, s)).cuda() for s in range(4)]
    return el, ii, oi, base


def bench_frame(base, k):
    import torch
    t = base[k % 4].clone()
    t[:: 4099] = (t[:: 4099].to(torch.int32) + k).to(torch.uint8)
    return t


def single(el, oi, frame):
    """the same frame alone on the same handle"""
    import torch
    dst = torch.full((oi.size,), vb.FILL, dtype=torch.uint8, device="cuda")
    el.transform_frame(frame, dst)
    torch.cuda.synchronize()
    return dst.cpu().numpy()


def test_headline_batch_on_a_stream(headline):
    """32 distinct frames per call, frames that share a base differing in a few pixels only: every output equals the
    frame converted alone, frames 0, 1, 4 and 31 equal the oracle, and no two outputs are the same"""
    import torch
    el, ii, oi, base = headline
    ins = [bench_frame(base, k) for k in range(FRAMES)]
    outs = [torch.full((oi.size,), vb.FILL, dtype=torch.uint8, device="cuda") for _ in range(FRAMES)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        el.transform_frames(ins, outs, stream)
    torch.cuda.synchronize()
    got = [o.cpu().numpy() for o in outs]
    assert len({hashlib.sha256(x.tobytes()).digest() for x in got}) == FRAMES, "two outputs of the batch are the same"
    for k in range(FRAMES):
        vb.same(got[k], single(el, oi, ins[k]), f"frame {k} of the batch vs alone")
    d = ob.vcs_desc(IW, IH, OW, OH, 3)
    for k in (0, 1, 4, 31):
        vb.same(got[k], ob.oracle_vcs_convert(d, ins[k].cpu().numpy()), f"frame {k} vs oracle")


def test_headline_host_frames(headline):
    """64 pinned frames through transform_host_frames (4-frame chunks through the staging ring): every output equals the
    frame converted alone on the device, frames 0 and 63 equal the oracle"""
    import torch
    import gstreamer_b200 as g
    el, ii, oi, base = headline
    n = 64
    hin = [g.PinnedBuffer(ii.size) for _ in range(n)]
    hout = [g.PinnedBuffer(oi.size) for _ in range(n)]
    try:
        for k, b in enumerate(hin):
            b.array[:] = bench_frame(base, k).cpu().numpy()
        for b in hout:
            b.array.fill(vb.FILL)
        el.transform_host_frames([b.ptr for b in hin], [b.ptr for b in hout])
        seen = set()
        for k in range(n):
            got = hout[k].array.copy()
            seen.add(hashlib.sha256(got.tobytes()).digest())
            vb.same(got, single(el, oi, torch.from_numpy(hin[k].array).cuda()), f"host frame {k} vs alone")
        assert len(seen) == n, "two outputs of the host call are the same"
        d = ob.vcs_desc(IW, IH, OW, OH, 3)
        for k in (0, n - 1):
            vb.same(hout[k].array, ob.oracle_vcs_convert(d, hin[k].array), f"host frame {k} vs oracle")
    finally:
        for b in hin + hout:
            b.free()
