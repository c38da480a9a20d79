#!/usr/bin/env python
"""tests/golden/make_host_staging.py — writes tests/golden/host_staging.json: what the system-memory ("host") entry
points issue, call by call.

Each record runs a short sequence of calls on handles it creates and holds each call's status (and output frame count
where the call reports one) and the emulated library's level-3 log (tests/cudaemu): every kernel launch and, between
them, each cudaMalloc / cudaFree, async copy and memset, event record, stream wait, synchronise, and stream or event
creation and destruction.  Handles and allocations are named by creation order, so the log holds no addresses.

- converter: b200_vcs_copy_probe, then b200_vcs_convert_host with n = 1, 2, 31, 32, 63, 64, 65, 130, 1 (the chunk grows
  1 -> 2 -> 4, a call follows a larger one, more chunks than slots), b200_vcs_copy_probe again, for two format pairs;
- compositor, packed RGB and NV12 / I420 / Y444 / I422_10LE output: more submissions than slots, b200_comp_blend_host_wait
  with keep 0 / 1 / 2 / 3, pads and destination growing between submissions, pads at alpha 0, at a negative alpha and
  SOURCE at alpha 0, destroy with submissions in flight;
- resampler, F32 and S16: waits before any submit, buffers that grow past and stay under the 25 % headroom, a drain
  (no input), keep 0..3, destroy with submissions in flight;
- the invalid arguments of every host entry point, and handles without a device.

    python tests/golden/make_host_staging.py        # rewrite the fixture
"""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "cudaemu"))
FIXTURE = os.path.join(HERE, "host_staging.json")

NV12, I420, Y444, I422_10LE, BGRA, RGBA = 23, 2, 20, 45, 12, 11
F32, S16 = 28, 4
SOURCE, OVER = 0, 1
CONVERTS = [1, 2, 31, 32, 63, 64, 65, 130, 1]
# (input format, width, height) -> (output format, width, height)
VCS_PAIRS = [((NV12, 64, 36), (BGRA, 32, 18)), ((I420, 40, 30), (NV12, 40, 30))]
COMP_YUV = [NV12, I420, Y444, I422_10LE]


def load():
    import build_emu
    from gstreamer_b200 import _lib
    lib = C.CDLL(build_emu.build())
    for name, (res, args) in _lib._SIGS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    lib.b200emu_launch_log.restype = C.c_char_p
    lib.b200emu_set_record_only.argtypes = [C.c_int]
    lib.b200emu_fail_create.argtypes = [C.c_int]
    return lib, _lib


class Host:
    """system memory of one record: numpy buffers kept alive, addressed by pointer"""

    def __init__(self, seed=0):
        self.keep, self.rng = [], np.random.default_rng(seed)

    def buf(self, nbytes):
        a = self.rng.integers(0, 256, max(nbytes, 1), dtype=np.uint8)
        self.keep.append(a)
        return a

    def ptrs(self, bufs):
        return (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs])


class Emu:
    def __init__(self):
        self.lib, self.c = load()

    def info(self, fmt, w, h, pad=0):
        """a frame's layout; `pad` adds bytes to every plane's stride"""
        i = self.c.VideoInfoC()
        assert self.lib.b200_video_info_set_format(C.byref(i), fmt, w, h) == 0
        if pad:
            n = sum(1 for s in i.stride if s)
            off = 0
            for p in range(n):
                rows = (i.offset[p + 1] - i.offset[p]) // i.stride[p] if p + 1 < n else \
                    (self.lib.b200_video_info_size(C.byref(i)) - i.offset[p]) // i.stride[p]
                i.stride[p] += pad
                i.offset[p] = off
                off += rows * i.stride[p]
        return i

    def size(self, info):
        return self.lib.b200_video_info_size(C.byref(info))

    def record(self, fn):
        """fn's results and the level-3 log of everything it issued"""
        self.lib.b200emu_clear_launch_log()
        self.lib.b200emu_set_record_only(3)
        try:
            out = fn()
        finally:
            self.lib.b200emu_set_record_only(0)
        log = self.lib.b200emu_launch_log().decode()
        self.lib.b200emu_clear_launch_log()
        return {"calls": out, "log": [x for x in log.split("\n") if x]}

    # ---- handles
    def vcs(self, pair, device=0):
        (fi, wi, hi), (fo, wo, ho) = pair
        ii, oi = self.info(fi, wi, hi), self.info(fo, wo, ho)
        h = C.c_void_p()
        assert self.lib.b200_vcs_create(C.byref(ii), C.byref(oi), None, device, C.byref(h)) == 0
        return h, self.size(ii), self.size(oi)

    def comp(self, fmt, w, h, device=0):
        hd = C.c_void_p()
        assert self.lib.b200_comp_create(fmt, w, h, device, C.byref(hd)) == 0
        return hd

    def ars(self, fmt, device=0, rates=(48000, 44100), channels=2):
        cfg = self.c.ArsConfigC()
        cfg.in_rate, cfg.out_rate = rates
        cfg.channels, cfg.format, cfg.quality = channels, fmt, 4
        h = C.c_void_p()
        assert self.lib.b200_ars_create(C.byref(cfg), device, C.byref(h)) == 0
        return h

    # ---- calls
    def convert_host(self, h, mem, n, in_bytes, out_bytes):
        ins = [mem.buf(in_bytes) for _ in range(n)]
        outs = [mem.buf(out_bytes) for _ in range(n)]
        return self.lib.b200_vcs_convert_host(h, n, mem.ptrs(ins), mem.ptrs(outs)), ins, outs

    def copy_probe(self, h, mem, n, in_bytes, out_bytes):
        ins = [mem.buf(in_bytes) for _ in range(n)]
        outs = [mem.buf(out_bytes) for _ in range(n)]
        return self.lib.b200_vcs_copy_probe(h, n, mem.ptrs(ins), mem.ptrs(outs))

    def rgb_pads(self, mem, specs):
        """specs: (width, height, stride padding, xpos, ypos, alpha, op)"""
        pads = (self.c.CompPadC * max(len(specs), 1))()
        for p, (w, h, sp, x, y, a, op) in zip(pads, specs):
            stride = w * 4 + sp
            p.data, p.width, p.height, p.stride = mem.buf(stride * h).ctypes.data, w, h, stride
            p.xpos, p.ypos, p.alpha, p.op = x, y, a, op
        return pads

    def yuv_pads(self, mem, fmt, specs):
        """specs: (width, height, stride padding, xpos, ypos, alpha, op)"""
        pads = (self.c.CompPadYuvC * max(len(specs), 1))()
        for p, (w, h, sp, x, y, a, op) in zip(pads, specs):
            p.info = self.info(fmt, w, h, sp)
            p.data = mem.buf(self.size(p.info)).ctypes.data
            p.xpos, p.ypos, p.alpha, p.op = x, y, a, op
        return pads

    def ars_submit(self, h, mem, n, bpf, cap=None, silent=False):
        want = self.lib.b200_ars_get_out_frames(h, n)
        cap = want if cap is None else cap
        src = None if silent else mem.buf(n * bpf).ctypes.data
        out = mem.buf(max(cap, 1) * bpf)
        got = C.c_size_t(12345)
        st = self.lib.b200_ars_process_host_submit(h, src, n, out.ctypes.data, cap, C.byref(got))
        return [st, got.value]


# pads of the compositor records: small, then larger (the slot's pad buffer grows), then the alpha classes
RGB_STEPS = [
    [(8, 6, 0, 1, 2, 1.0, OVER), (6, 4, 4, 20, 10, 0.5, OVER)],
    [(8, 6, 0, 1, 2, 1.0, OVER)],
    [(8, 6, 0, 3, 3, 0.7, OVER), (10, 8, 8, 9, 1, 1.0, OVER)],
    [(16, 12, 0, -3, -2, 1.0, OVER), (12, 10, 4, 20, 20, 0.25, OVER)],
    [(8, 6, 0, 0, 0, 0.0, OVER), (8, 6, 0, 4, 4, -0.5, OVER), (8, 6, 0, 8, 8, 0.0, SOURCE), (6, 6, 0, 2, 2, 0.5, OVER)],
    [(20, 16, 0, 5, 5, 0.8, OVER)],
]


def rec_vcs(e, pair):
    def run():
        mem = Host(1)
        h, ib, ob = e.vcs(pair)
        out = [e.copy_probe(h, mem, 3, ib, ob)]
        for n in CONVERTS:
            out.append(e.convert_host(h, mem, n, ib, ob)[0])
        out.append(e.copy_probe(h, mem, 5, ib, ob))
        e.lib.b200_vcs_destroy(h)
        return out
    return e.record(run)


def rec_comp_rgb(e):
    def run():
        mem = Host(2)
        W, H = 32, 24
        h = e.comp(BGRA, W, H)
        out = [e.lib.b200_comp_blend_host_wait(h, 0), e.lib.b200_comp_blend_host_wait(h, 3)]
        waits = {1: 2, 3: 1, 4: 0, 5: 3}
        for k, specs in enumerate(RGB_STEPS):
            stride = W * 4 + (64 if k >= 3 else 0)                     # the destination grows from the fourth frame on
            dst = mem.buf(stride * H)
            out.append(e.lib.b200_comp_blend_host_submit(h, dst.ctypes.data, stride, k % 4, e.rgb_pads(mem, specs), len(specs)))
            if k in waits:
                out.append(e.lib.b200_comp_blend_host_wait(h, waits[k]))
        dst = mem.buf(W * 4 * H)
        out.append(e.lib.b200_comp_blend_host(h, dst.ctypes.data, W * 4, 0, e.rgb_pads(mem, RGB_STEPS[0]), 2))
        out.append(e.lib.b200_comp_blend_host_submit(h, dst.ctypes.data, W * 4, 1, e.rgb_pads(mem, RGB_STEPS[1]), 1))
        e.lib.b200_comp_destroy(h)                                     # one submission in flight
        return out
    return e.record(run)


def rec_comp_yuv(e, fmt):
    def run():
        mem = Host(3)
        W, H = 32, 24
        h = e.comp(fmt, W, H)
        out = [e.lib.b200_comp_blend_host_wait(h, 1)]
        waits = {1: 2, 3: 1, 4: 0, 5: 3}
        for k, specs in enumerate(RGB_STEPS):
            di = e.info(fmt, W, H, 16 if k >= 3 else 0)
            dst = mem.buf(e.size(di))
            out.append(e.lib.b200_comp_blend_yuv_host_submit(h, dst.ctypes.data, C.byref(di), k % 4,
                                                              e.yuv_pads(mem, fmt, specs), len(specs)))
            if k in waits:
                out.append(e.lib.b200_comp_blend_host_wait(h, waits[k]))
        di = e.info(fmt, W, H)
        dst = mem.buf(e.size(di))
        out.append(e.lib.b200_comp_blend_yuv_host(h, dst.ctypes.data, C.byref(di), 0, e.yuv_pads(mem, fmt, RGB_STEPS[0]), 2))
        out.append(e.lib.b200_comp_blend_yuv_host_submit(h, dst.ctypes.data, C.byref(di), 1, e.yuv_pads(mem, fmt, RGB_STEPS[1]), 1))
        e.lib.b200_comp_destroy(h)
        return out
    return e.record(run)


def rec_ars(e, fmt):
    def run():
        mem = Host(4)
        bpf = 2 * (4 if fmt == F32 else 2)
        h = e.ars(fmt)
        out = [e.lib.b200_ars_process_host_wait(h, 0), e.lib.b200_ars_process_host_wait(h, 3)]
        # slot 0: 480 frames, then 400 (under its capacity); slot 1: 960, then 1100 (under the headroom of 960);
        # slot 2: 1000, then 1300 (past it)
        for n, keep in ((480, None), (960, 2), (1000, None), (400, 1), (1100, None), (1300, 0), (200, 3)):
            out.append(e.ars_submit(h, mem, n, bpf, silent=n == 200))
            if keep is not None:
                out.append(e.lib.b200_ars_process_host_wait(h, keep))
        out.append(e.ars_submit(h, mem, 500, bpf, cap=3))                 # output capacity too small
        n = 700
        want = e.lib.b200_ars_get_out_frames(h, n)
        src, dst, got = mem.buf(n * bpf), mem.buf(want * bpf), C.c_size_t(0)
        out.append([e.lib.b200_ars_process_host(h, src.ctypes.data, n, dst.ctypes.data, want, C.byref(got)), got.value])
        out.append(e.ars_submit(h, mem, 300, bpf))
        e.lib.b200_ars_destroy(h)                                          # one submission in flight
        return out
    return e.record(run)


def rec_errors(e):
    def run():
        mem = Host(5)
        lib, out = e.lib, []
        h, ib, ob = e.vcs(VCS_PAIRS[0])
        ins, outs = mem.ptrs([mem.buf(ib)] * 2), mem.ptrs([mem.buf(ob)] * 2)
        holes = (C.c_void_p * 2)(ins[0], None)
        for fn in (lib.b200_vcs_convert_host, lib.b200_vcs_copy_probe):
            out += [fn(None, 2, ins, outs), fn(h, 2, None, outs), fn(h, 2, ins, None), fn(h, 0, ins, outs),
                    fn(h, -1, ins, outs), fn(h, 2, holes, outs), fn(h, 2, ins, holes)]
        lib.b200_vcs_destroy(h)
        hh, _, _ = e.vcs(VCS_PAIRS[0], device=-1)
        out += [lib.b200_vcs_convert_host(hh, 2, ins, outs), lib.b200_vcs_copy_probe(hh, 2, ins, outs)]
        lib.b200_vcs_destroy(hh)

        W, H = 32, 24
        rgb, yuv = e.comp(BGRA, W, H), e.comp(NV12, W, H)
        dst = mem.buf(W * 4 * H * 2).ctypes.data
        good = e.rgb_pads(mem, RGB_STEPS[0])
        sub = lib.b200_comp_blend_host_submit
        out += [sub(None, dst, W * 4, 0, good, 2), sub(rgb, None, W * 4, 0, good, 2), sub(rgb, dst, W * 4, 0, good, -1),
                sub(rgb, dst, W * 4, 0, good, 65), sub(rgb, dst, W * 4, 0, None, 1), sub(yuv, dst, W * 4, 0, good, 2),
                sub(rgb, dst, W * 4 - 4, 0, good, 2), sub(rgb, dst, W * 4 + 2, 0, good, 2)]
        for spec in ((8, 6, -4, 0, 0, 1.0, OVER), (0, 6, 0, 0, 0, 1.0, OVER), (8, 0, 0, 0, 0, 1.0, OVER)):
            out.append(sub(rgb, dst, W * 4, 0, e.rgb_pads(mem, [spec]), 1))
        nulled = e.rgb_pads(mem, RGB_STEPS[0][:1])
        nulled[0].data = None
        out.append(sub(rgb, dst, W * 4, 0, nulled, 1))
        di = e.info(NV12, W, H)
        ygood = e.yuv_pads(mem, NV12, RGB_STEPS[0])
        ysub = lib.b200_comp_blend_yuv_host_submit
        out += [ysub(None, dst, C.byref(di), 0, ygood, 2), ysub(yuv, None, C.byref(di), 0, ygood, 2),
                ysub(yuv, dst, None, 0, ygood, 2), ysub(yuv, dst, C.byref(di), 0, ygood, -1),
                ysub(yuv, dst, C.byref(di), 0, ygood, 65), ysub(yuv, dst, C.byref(di), 0, None, 1),
                ysub(rgb, dst, C.byref(di), 0, ygood, 2)]
        ybad = e.yuv_pads(mem, NV12, RGB_STEPS[0][:1])
        ybad[0].info.width = 0
        out.append(ysub(yuv, dst, C.byref(di), 0, ybad, 1))
        ybad = e.yuv_pads(mem, NV12, RGB_STEPS[0][:1])
        ybad[0].data = None
        out.append(ysub(yuv, dst, C.byref(di), 0, ybad, 1))
        wait = lib.b200_comp_blend_host_wait
        out += [wait(None, 0), wait(rgb, -1), wait(rgb, 3), wait(rgb, 2)]
        out.append(sub(rgb, dst, W * 4, 0, good, 2))
        out += [wait(rgb, 3), wait(rgb, 1), wait(rgb, 0)]
        lib.b200_comp_destroy(rgb)
        lib.b200_comp_destroy(yuv)
        ho = e.comp(BGRA, W, H, device=-1)
        out += [sub(ho, dst, W * 4, 0, good, 2), wait(ho, 0), wait(ho, -1)]
        lib.b200_comp_destroy(ho)
        ho = e.comp(NV12, W, H, device=-1)
        out += [ysub(ho, dst, C.byref(di), 0, ygood, 2)]
        lib.b200_comp_destroy(ho)

        h = e.ars(F32)
        src, dsta, got = mem.buf(4000).ctypes.data, mem.buf(4000).ctypes.data, C.c_size_t(7)
        asub, await_ = lib.b200_ars_process_host_submit, lib.b200_ars_process_host_wait
        out += [asub(None, src, 100, dsta, 500, C.byref(got)), asub(h, src, 100, None, 500, C.byref(got)),
                asub(h, src, 100, dsta, 1, C.byref(got)), asub(h, src, 100, dsta, 500, None),
                await_(None, 0), await_(h, -1), await_(h, 3), await_(h, 2), await_(h, 0)]
        lib.b200_ars_destroy(h)
        ho = e.ars(F32, device=-1)
        out += [asub(ho, src, 100, dsta, 500, C.byref(got)), await_(ho, 0), await_(ho, 3),
                lib.b200_ars_process_host(ho, src, 100, dsta, 500, C.byref(got))]
        lib.b200_ars_destroy(ho)
        return out
    return e.record(run)


def record():
    e = Emu()
    out = {}
    for pair in VCS_PAIRS:
        out["vcs %d>%d" % (pair[0][0], pair[1][0])] = rec_vcs(e, pair)
    out["comp rgb"] = rec_comp_rgb(e)
    for fmt in COMP_YUV:
        out["comp yuv %d" % fmt] = rec_comp_yuv(e, fmt)
    for fmt in (F32, S16):
        out["ars %d" % fmt] = rec_ars(e, fmt)
    out["errors"] = rec_errors(e)
    return out


if __name__ == "__main__":
    with open(FIXTURE, "w") as f:
        json.dump(record(), f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", FIXTURE)
