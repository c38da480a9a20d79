"""TEST INFRASTRUCTURE: the converter's batch routes (b200_vcs_convert_batch), shared by tests/test_vcs_batch_gpu.py (the
H100) and tests/test_emu_batch.py (the emulated library, tests/cudaemu).

Each row is one handle configuration and the launch sequence it must produce; together the rows launch every kernel a
convert can reach.  The checks run a row's handle on batches of distinct frames and compare every output with its own
frame's expected bytes: a kernel that took its frame from the wrong batch slot, or a chain whose frames shared one
slice of the scratch image, fails them.  They take the library (ctypes, the b200_vcs_* C-ABI) and a memory backend
(HostMem here, device memory in the GPU file) so that the same code runs on the H100 and on the emulator."""
import ctypes as C
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np

from oracle import bindings as ob
from rgbp_oracle import FMT, oracle_rgbp

MAX_BATCH = 64                                     # B200_VCS_MAX_BATCH
ERR_INVALID_ARG = -1                               # B200_ERR_INVALID_ARG
FILL = 0x5A                                        # output bytes a conversion does not write keep it
GUARD = 4096                                       # bytes around each frame of the unordered arenas
BORDER = 0xff204060                                # border colour of the destination-rectangle rows
YUV420 = ("NV12", "NV21", "I420", "YV12")
YUV_422_444 = ("YUY2", "UYVY", "YVYU", "Y42B", "Y444")


@dataclass(frozen=True)
class Row:
    id: str
    fi: str
    fo: str
    size: Tuple[int, int, int, int]                # iw, ih, ow, oh
    method: int
    name: str                                      # b200_vcs_kernel_name
    launches: Tuple[str, ...]                      # the launch sequence, as the emulated library logs it
    site: Optional[int] = None                     # the input's chroma site (None: the default of its size)
    pillar: bool = False                           # the element's add-borders rectangle (a pillar box), BORDER around it
    variant: Optional[int] = None                  # b200_vcs_set_kernel_variant after create
    knob: Optional[str] = None                     # "NAME=value", set before the handle is created
    device_only: bool = False                      # vcs_l2tc_kernel (wgmma) is not in the emulated library


ROWS = [
    # the exact 2:1 / 8-tap kernels; chroma site 2 (MPEG-2) is what makes these shapes eligible
    Row("nv12-bgra-2to1", "NV12", "BGRA", (256, 144, 128, 72), 3, "vcs_lanczos2_v2_kernel",
        ("vcs_lanczos2_v2_kernel<4, 291, 0, 60, 256, false, false, false>",), site=2),
    Row("i420-bgra-2to1", "I420", "BGRA", (256, 144, 128, 72), 3, "vcs_lanczos2_v2_kernel",
        ("vcs_lanczos2_v2_kernel<4, 291, 0, 60, 256, true, false, false>",), site=2),
    Row("nv12-rgba-2to1-v1", "NV12", "RGBA", (256, 144, 128, 72), 3, "vcs_lanczos2_kernel",
        ("vcs_lanczos2_kernel<true, 4, 60, 1, true>",), site=2, knob="B200_L2_V1=1"),
    Row("nv12-bgra-2to1-mma", "NV12", "BGRA", (256, 144, 128, 72), 3, "vcs_l2mma_kernel", ("vcs_l2mma_kernel",), site=2, variant=6),
    Row("nv12-bgra-2to1-tc", "NV12", "BGRA", (256, 144, 128, 72), 3, "vcs_l2tc_kernel", ("vcs_l2tc_kernel",), site=2, variant=7,
        device_only=True),
    # the other kernels into packed RGB
    Row("nv12-bgra-light", "NV12", "BGRA", (200, 120, 133, 80), 1, "vcs_light_kernel", ("vcs_light_kernel<2, 2, false, false, false>",)),
    Row("nv12-bgra-ntap", "NV12", "BGRA", (96, 54, 64, 36), 3, "vcs_ntap_kernel", ("vcs_ntap_kernel<3, 3, false, false, 2, false>",)),
    Row("nv12-bgra-ntap-vfirst", "NV12", "BGRA", (100, 60, 150, 30), 3, "vcs_ntap_kernel",
        ("vcs_ntap_vfirst_kernel<3, 3, false, false, false>",)),
    Row("y444-bgra-generic", "Y444", "BGRA", (64, 48, 40, 30), 1, "vcs_generic_kernel", ("vcs_generic_kernel<false>",)),
    Row("nv12-bgra-pillar", "NV12", "BGRA", (96, 96, 160, 90), 1, "vcs_light_kernel",
        ("vcs_border_kernel", "vcs_light_kernel<2, 2, false, false, false>"), pillar=True),
    # 4:2:0 -> the other 4:2:0 family: the scaled pixels of every frame into its slice of the scratch image, then
    # vcs_down420_kernel
    Row("nv12-i420-2to1", "NV12", "I420", (256, 144, 128, 72), 3, "vcs_lanczos2_v2_kernel",
        ("vcs_lanczos2_v2_kernel<4, -1, 0, 60, 256, false, true, false>", "vcs_down420_kernel"), site=2),
    Row("nv12-i420-ntap", "NV12", "I420", (100, 60, 64, 36), 3, "vcs_ntap_kernel",
        ("vcs_ntap_vfirst_kernel<3, 3, false, false, false>", "vcs_down420_kernel")),
    Row("nv12-i420-generic", "NV12", "I420", (100, 60, 64, 36), 3, "vcs_ntap_kernel",
        ("vcs_generic_kernel<false>", "vcs_down420_kernel"), knob="B200_CROSS_GENERIC=1"),
    Row("nv12-i420-odd-height", "NV12", "I420", (64, 49, 32, 49), 1, "vcs_light_kernel",   # scratch row oh: generic kernel
        ("vcs_light_kernel<2, 1, false, false, false>", "vcs_generic_kernel<false>", "vcs_down420_kernel")),
    # packed RGB / packed 4:2:2 -> 4:2:0
    Row("bgra-nv12-same", "BGRA", "NV12", (64, 48, 64, 48), 1, "vcs_rgb420_kernel", ("vcs_rgb420_kernel<true>",)),
    Row("rgba-i420-down", "RGBA", "I420", (100, 60, 64, 36), 3, "vcs_rgb420_kernel",
        ("vcs_planes_fast_vfirst_kernel<3, 3, 4, 2>", "vcs_rgb420_kernel<true>")),
    Row("xrgb-nv21-up", "xRGB", "NV21", (40, 30, 64, 48), 1, "vcs_rgb420_kernel",
        ("vcs_rgb2ayuv_kernel", "vcs_planes_fast_kernel<2, 2, 4, 0>", "vcs_rgb420_kernel<false>")),
    Row("bgra-nv12-generic", "BGRA", "NV12", (100, 60, 64, 36), 1, "vcs_generic_kernel",
        ("vcs_generic_kernel<false>", "vcs_down420_kernel"), knob="B200_RGB420_GENERIC=1"),
    Row("yuy2-i420-same", "YUY2", "I420", (64, 48, 64, 48), 1, "vcs_yuy2_420_kernel", ("vcs_yuy2_420_kernel",)),
    Row("yuy2-nv12-down", "YUY2", "NV12", (100, 60, 64, 36), 1, "vcs_yuy2_ayuv_kernel",
        ("vcs_yuy2_ayuv_kernel", "vcs_planes_fast_vfirst_kernel<2, 2, 4, 0>", "vcs_rgb420_kernel<false>")),
    # same-family plane scaling
    Row("nv12-nv12-slow", "NV12", "NV12", (100, 60, 64, 36), 3, "vcs_planes_kernel", ("vcs_planes_kernel",), knob="B200_PLANES_SLOW=1"),
    Row("nv12-nv12-fast", "NV12", "NV12", (96, 200, 96, 75), 3, "vcs_planes_fast_kernel",
        ("vcs_planes_fast_kernel<1, 3, 1, 0>", "vcs_planes_fast_kernel<1, 3, 2, 0>")),
    Row("i420-yv12-vfirst", "I420", "YV12", (100, 60, 64, 36), 3, "vcs_planes_fast_vfirst_kernel",
        ("vcs_planes_fast_vfirst_kernel<3, 3, 1, 2>", "vcs_planes_fast_vfirst_kernel<3, 3, 1, 1>", "vcs_planes_fast_vfirst_kernel<3, 3, 1, 1>")),
    Row("nv21-nv21-halve", "NV21", "NV21", (128, 64, 64, 32), 1, "vcs_planes_fast_vfirst_kernel",
        ("vcs_planes_vec_kernel", "vcs_planes_fast_vfirst_kernel<3, 2, 2, 1>")),
    Row("i420-i420-copy", "I420", "I420", (64, 48, 64, 48), 1, "vcs_planes_kernel",
        ("vcs_planes_vec_kernel", "vcs_planes_vec_kernel", "vcs_planes_vec_kernel")),
    Row("i420-i420-pillar", "I420", "I420", (96, 96, 160, 90), 1, "vcs_planes_fast_vfirst_kernel",
        ("vcs_border_kernel",) + ("vcs_planes_fast_vfirst_kernel<2, 2, 1, 0>",) * 3, pillar=True),
    # packed RGB -> planar RGB at an unchanged size: the de-interleave alone, reading the frames themselves
    Row("bgra-rgbp-same", "BGRA", "RGBP", (64, 48, 64, 48), 1, "vcs_rgb_deinterleave_kernel", ("vcs_rgb_deinterleave_kernel",)),
]


def kernels(rows):
    """the kernels the rows launch, template arguments dropped"""
    return {x.split("<")[0] for r in rows for x in r.launches}


# ---- one handle -----------------------------------------------------------------------------------------------------
class Handle:
    """b200_vcs_create of a row on `lib` (the product's library or the emulated one), with the row's knob and variant"""

    def __init__(self, lib, row, monkeypatch, device=0):
        from gstreamer_b200 import _lib
        if row.knob:
            monkeypatch.setenv(*row.knob.split("="))       # read by b200_vcs_create
        self.lib, self.row = lib, row
        iw, ih, ow, oh = row.size
        self.ii, self.oi = _lib.VideoInfoC(), _lib.VideoInfoC()
        assert lib.b200_video_info_set_format(C.byref(self.ii), FMT[row.fi], iw, ih) == 0
        assert lib.b200_video_info_set_format(C.byref(self.oi), FMT[row.fo], ow, oh) == 0
        if row.site is not None:
            self.ii.chroma_site = row.site
        if row.fi in YUV420 and row.fo in YUV420:           # what the element's caps fixation does
            self.oi.color_matrix, self.oi.color_range, self.oi.chroma_site = self.ii.color_matrix, self.ii.color_range, self.ii.chroma_site
        elif row.fi in YUV_422_444 and row.fo in YUV420:    # ... across a sub-sampling change: the site stays the output's own
            self.oi.color_matrix, self.oi.color_range = self.ii.color_matrix, self.ii.color_range
        cfg = _lib.VcsConfigC()
        lib.b200_vcs_config_init(C.byref(cfg))
        cfg.method = row.method
        self.dest = None
        if row.pillar:
            self.dest = ob.vcs_borders(*row.size)
            assert self.dest[1] == 0 and self.dest[3] == oh and self.dest[2] < ow, ("not a pillar box", self.dest)
            cfg.dest_x, cfg.dest_y, cfg.dest_width, cfg.dest_height = self.dest
            cfg.border_argb = BORDER
        self.h = C.c_void_p()
        assert lib.b200_vcs_create(C.byref(self.ii), C.byref(self.oi), C.byref(cfg), device, C.byref(self.h)) == 0, row
        if row.variant is not None:
            assert lib.b200_vcs_set_kernel_variant(self.h, row.variant) == 0, "variant %d not eligible" % row.variant
        self.in_size = lib.b200_video_info_size(C.byref(self.ii))
        self.out_size = lib.b200_video_info_size(C.byref(self.oi))
        info = _lib.VcsPlanInfoC()
        assert lib.b200_vcs_get_plan_info(self.h, C.byref(info)) == 0
        # the handle's own account of its route, before the row trusts its label
        assert lib.b200_vcs_kernel_name(self.h).decode() == row.name, (row.id, lib.b200_vcs_kernel_name(self.h))
        assert info.n_launches_per_convert == len(row.launches), (row.id, info.n_launches_per_convert)
        if row.variant is not None:
            assert info.kernel_variant == row.variant

    def convert(self, ins, outs, stream=None):
        n = len(ins)
        a = (C.c_void_p * max(n, 1))(*ins)
        b = (C.c_void_p * max(n, 1))(*outs)
        return self.lib.b200_vcs_convert_batch(self.h, n, a, b, stream)

    def close(self):
        if self.h:
            self.lib.b200_vcs_destroy(self.h)
            self.h = None

    # ---- frames and what they must become ------------------------------------------------------------------------
    def frame(self, seed):
        """a random input frame of the row's format and default layout"""
        return np.random.default_rng(seed).integers(0, 256, self.in_size, dtype=np.uint8)

    def expected(self, frame):
        """the whole output buffer: the oracle's pixel bytes, FILL in row padding and between planes"""
        r = self.row
        iw, ih, ow, oh = r.size
        if r.fo in ("RGBP", "BGRP"):
            layout = ([self.oi.stride[k] for k in range(3)], [self.oi.offset[k] for k in range(3)])
            return oracle_rgbp(r.fi, r.fo, r.size, r.method, frame, site=r.site, layout=layout, dest=self.dest, border=BORDER, fill=FILL)
        d = ob.vcs_desc(iw, ih, ow, oh, r.method, in_fmt=FMT[r.fi], out_fmt=FMT[r.fo], site=r.site)
        isz, osz = ob.vcs_sizes(d)
        assert isz <= frame.size and osz == self.out_size
        if self.dest:
            return ob.oracle_vcs_convert_dest(d, frame, self.dest, BORDER, fill=FILL)
        want = ob.oracle_vcs_convert(d, frame)
        if r.fo not in YUV420:
            return want
        out = np.full(self.out_size, FILL, dtype=np.uint8)
        semi = r.fo in ("NV12", "NV21")
        for p in range(2 if semi else 3):
            w = ow if p == 0 else ((ow + 1) // 2) * (2 if semi else 1)
            h = oh if p == 0 else (oh + 1) // 2
            st, off = self.oi.stride[p], self.oi.offset[p]
            out[off: off + st * h].reshape(h, st)[:, :w] = want[off: off + st * h].reshape(h, st)[:, :w]
        return out


def distinct(wants, tag):
    """the batch's power: outputs that all differ, so that a frame read from or written to another slot shows"""
    assert len({w.tobytes() for w in wants}) == len(wants), f"{tag}: expected outputs of the batch are not pairwise different"


def same(got, want, tag):
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{tag}: {bad.size} of {got.size} bytes differ, first at {bad[:6].tolist()}"


# ---- memory -----------------------------------------------------------------------------------------------------------
class HostMem:
    """the emulated library's "device memory": host arrays, each starting on a 256-byte boundary"""
    stream = None

    def buffer(self, nbytes):
        raw = np.full(nbytes + 256, FILL, dtype=np.uint8)
        off = (-raw.ctypes.data) % 256
        return raw[off: off + nbytes]

    def ptr(self, b):
        return b.ctypes.data

    def put(self, b, off, data):
        b[off: off + data.size] = data

    def get(self, b):
        return b.copy()

    def sync(self):
        pass


# ---- the checks ---------------------------------------------------------------------------------------------------------
def check_batches(h, mem, sizes, seed):
    """one handle, a batch of new distinct frames per call at each of `sizes` (growing and shrinking: the scratch image is
    reallocated and its slices reused); every output equals its own frame's expected buffer"""
    for call, n in enumerate(sizes):
        frames = [h.frame(seed + 1000 * call + k) for k in range(n)]
        wants = [h.expected(f) for f in frames]
        distinct(wants, f"{h.row.id} n={n}")
        ins, outs = [mem.buffer(h.in_size) for _ in range(n)], [mem.buffer(h.out_size) for _ in range(n)]
        for b, f in zip(ins, frames):
            mem.put(b, 0, f)
        assert h.convert([mem.ptr(b) for b in ins], [mem.ptr(b) for b in outs], mem.stream) == 0
        mem.sync()
        for k in range(n):
            same(mem.get(outs[k]), wants[k], f"{h.row.id} call {call} (n={n}) frame {k}")


def _arena(mem, size, n, order):
    """one allocation holding n frames of `size` bytes, frame i in slot order[i], GUARD bytes around every slot"""
    slot = ((size + 255) & ~255) + GUARD
    buf = mem.buffer(GUARD + n * slot)
    offs = [GUARD + int(order[i]) * slot for i in range(n)]
    return buf, offs


def check_unordered(h, mem, n, seed):
    """all inputs in one allocation and all outputs in another, at shuffled offsets with guards between them: the batch's
    pointers neither increase nor step by a frame size.  Guards and inputs come back untouched."""
    rng = np.random.default_rng(seed)
    frames = [h.frame(seed + k) for k in range(n)]
    wants = [h.expected(f) for f in frames]
    distinct(wants, f"{h.row.id} unordered")
    while True:
        oi, oo = rng.permutation(n), rng.permutation(n)
        steps = {int(oi[k + 1]) - int(oi[k]) for k in range(n - 1)} | {int(oo[k + 1]) - int(oo[k]) for k in range(n - 1)}
        if len(steps) > 1 and not (oi == oo).all():
            break
    ib, ioffs = _arena(mem, h.in_size, n, oi)
    ob_, ooffs = _arena(mem, h.out_size, n, oo)
    for f, off in zip(frames, ioffs):
        mem.put(ib, off, f)
    assert all(off % 256 == 0 for off in ioffs + ooffs)
    before = mem.get(ib)
    base_i, base_o = mem.ptr(ib), mem.ptr(ob_)
    assert h.convert([base_i + o for o in ioffs], [base_o + o for o in ooffs], mem.stream) == 0
    mem.sync()
    got = mem.get(ob_)
    written = np.zeros(got.size, dtype=bool)
    for k, off in enumerate(ooffs):
        same(got[off: off + h.out_size], wants[k], f"{h.row.id} unordered frame {k} (slot {oo[k]})")
        written[off: off + h.out_size] = True
    assert (got[~written] == FILL).all(), f"{h.row.id}: a guard of the output arena was written"
    same(mem.get(ib), before, f"{h.row.id}: input arena")


def check_aliased_input(h, mem, seed):
    """one input twice in the batch, each time to its own output"""
    a, b = h.frame(seed), h.frame(seed + 1)
    wa, wb = h.expected(a), h.expected(b)
    distinct([wa, wb], f"{h.row.id} aliased")
    ia, ib = mem.buffer(h.in_size), mem.buffer(h.in_size)
    mem.put(ia, 0, a)
    mem.put(ib, 0, b)
    outs = [mem.buffer(h.out_size) for _ in range(3)]
    assert h.convert([mem.ptr(ia), mem.ptr(ib), mem.ptr(ia)], [mem.ptr(o) for o in outs], mem.stream) == 0
    mem.sync()
    for k, w in enumerate((wa, wb, wa)):
        same(mem.get(outs[k]), w, f"{h.row.id} aliased-input batch frame {k}")


def check_too_many(h, mem, seed):
    """MAX_BATCH + 1 frames: refused, nothing written"""
    src = mem.buffer(h.in_size)
    mem.put(src, 0, h.frame(seed))
    out, offs = _arena(mem, h.out_size, MAX_BATCH + 1, list(range(MAX_BATCH + 1)))
    assert h.convert([mem.ptr(src)] * (MAX_BATCH + 1), [mem.ptr(out) + o for o in offs], mem.stream) == ERR_INVALID_ARG
    mem.sync()
    assert (mem.get(out) == FILL).all(), f"{h.row.id}: a refused batch wrote output bytes"
