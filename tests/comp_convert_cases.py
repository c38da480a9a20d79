"""Cases for b200_comp_blend_convert and their expected bytes (tests/test_comp_convert.py on the emulated library,
tests/test_comp_convert_gpu.py on the device).  Expected bytes come from existing code only: each converted pad through
oracle_vcs_convert (method 9, mitchell; the pad's input -> the output format at the pad's output size), then
oracle_compositor / oracle_compositor_yuv at the pad's position."""
import ctypes as C

import numpy as np

from oracle import bindings as ob

FMT = dict(ob.FMT, I420=2, YV12=3, YUY2=4, NV12=23, NV21=24, Y444=20)
YUV420 = ("I420", "YV12", "NV12", "NV21")
IN_FORMATS = ("NV12", "NV21", "I420", "YV12", "YUY2", "Y444", "BGRx")
ALPHAS = (0.0, 0.004, 0.5, 0.999, 1.0)
MITCHELL = 9


def geometry(name, w, h):
    """(bytes per row, rows) of every plane"""
    cw, ch = (w + 1) // 2, (h + 1) // 2
    if name in ("NV12", "NV21"):
        return [(w, h), (2 * cw, ch)]
    if name in ("I420", "YV12"):
        return [(w, h), (cw, ch), (cw, ch)]
    if name == "Y444":
        return [(w, h)] * 3
    if name == "YUY2":
        return [(4 * cw, h)]
    return [(4 * w, h)]


def info(lib, name, w, h, odd=False):
    """the default layout; odd=True: rows at strides and planes at offsets that are not multiples of 4 (packed RGB keeps
    whole pixels: strides and offsets of 4-byte multiples that are not multiples of 16); odd="pitch": GstCudaMemory's
    layout, one pitch for every plane and planes at pitch-aligned offsets"""
    from gstreamer_b200 import _lib
    i = _lib.VideoInfoC()
    assert lib.b200_video_info_set_format(C.byref(i), FMT[name], w, h) == 0
    if odd == "pitch":
        pitch, off = 512, 0
        for k, (_, rows) in enumerate(geometry(name, w, h)):
            i.stride[k], i.offset[k] = pitch, off
            off += pitch * ((rows + 15) // 16 * 16)
    elif odd:
        rgb = len(geometry(name, w, h)) == 1 and name != "YUY2"
        off = 4 if rgb else 3
        for k, (rb, rows) in enumerate(geometry(name, w, h)):
            i.stride[k] = rb + (12 if rgb else 5 + 2 * k)
            i.offset[k] = off
            off += i.stride[k] * rows + (4 if rgb else 1)
    return i


def frame_size(name, i):
    return max(i.offset[k] + i.stride[k] * rows for k, (_, rows) in enumerate(geometry(name, i.width, i.height)))


def pack(name, a, i, fill=0x5A):
    """the planes' bytes `a` (rows back to back) laid out as `i`"""
    out = np.full(frame_size(name, i), fill, dtype=np.uint8)
    pos = 0
    for k, (rb, rows) in enumerate(geometry(name, i.width, i.height)):
        plane = a[pos: pos + rb * rows].reshape(rows, rb)
        pos += rb * rows
        view = out[i.offset[k]: i.offset[k] + i.stride[k] * rows].reshape(rows, i.stride[k])
        view[:, :rb] = plane
    return out


def unpack(name, buf, i):
    parts = []
    for k, (rb, rows) in enumerate(geometry(name, i.width, i.height)):
        parts.append(buf[i.offset[k]: i.offset[k] + i.stride[k] * rows].reshape(rows, i.stride[k])[:, :rb].reshape(-1))
    return np.concatenate(parts)


def random_frame(lib, name, w, h, seed):
    """a frame in the default layout (what the oracle reads), random bytes"""
    return np.random.default_rng(seed).integers(0, 256, frame_size(name, info(lib, name, w, h)), dtype=np.uint8)


def pad(in_fmt, iw, ih, pw, ph, x, y, alpha=1.0, op=1, seed=0, odd=False, kar=False):
    return dict(in_fmt=in_fmt, iw=iw, ih=ih, pw=pw, ph=ph, x=x, y=y, alpha=alpha, op=op, seed=seed, odd=odd, kar=kar)


def random_case(rng, out, trial, max_size, max_pads, min_pads=0, pad_max=None):
    W, H = (int(rng.integers(max(2, m // 3), m + 1)) for m in max_size)
    n = int(rng.integers(min_pads, max_pads + 1))
    pads, shared = [], []
    for i in range(n):
        if shared and rng.random() < 0.3:                           # the same conversion as an earlier pad
            p = dict(shared[int(rng.integers(0, len(shared)))])
        else:
            kind = rng.random()
            if out in YUV420:
                fmt = out if kind < 0.55 else str(rng.choice(IN_FORMATS))
            else:
                fmt = str(rng.choice(IN_FORMATS + (out,) * 3))
            pm = pad_max or (W + 8, H + 8)
            iw, ih = int(rng.integers(2, pm[0] + 1)), int(rng.integers(2, pm[1] + 1))
            if fmt == out and rng.random() < 0.3:
                pw, ph = iw, ih                                      # no conversion: the blend kernel's pad
            else:
                pw, ph = int(rng.integers(1, pm[0] + 1)), int(rng.integers(1, pm[1] + 1))
            odd = fmt == out and rng.random() < 0.5
            p = pad(fmt, iw, ih, pw, ph, 0, 0, seed=int(rng.integers(1 << 30)), odd=odd, kar=rng.random() < 0.15)
            if p["kar"] and 0 in output_size(p)[:2]:                # no picture left: the aggregator has nothing to convert
                p["kar"] = False
            shared.append(p)
        p = dict(p)
        p["x"] = int(rng.integers(-p["pw"] - 2, W + 2))
        p["y"] = int(rng.integers(-p["ph"] - 2, H + 2))
        p["alpha"] = float(rng.choice(ALPHAS))
        p["op"] = int(rng.integers(0, 3))
        pads.append(p)
    return dict(out=out, W=W, H=H, bg=int(trial % 4), dst_odd=trial % 2 == 1, pads=pads)


def mosaic_case(out, tile, src, grid, in_fmt=None):
    tw, th = tile
    pads = [pad(in_fmt or out, src[0], src[1], tw, th, c * tw, r * th, seed=1 + r * grid[0] + c)
            for r in range(grid[1]) for c in range(grid[0])]
    return dict(out=out, W=tw * grid[0], H=th * grid[1], bg=1, dst_odd=False, pads=pads)


def conv_launches(lib, case):
    """the launches of one convert by the first pad's converter (its plane kernels)"""
    from gstreamer_b200 import _lib
    s = Setup(lib, EmptyMem(), case)
    try:
        pi = _lib.VcsPlanInfoC()
        assert lib.b200_vcs_get_plan_info(s.pads[0].conv, C.byref(pi)) == 0
        return pi.n_launches_per_convert
    finally:
        s.close()


def output_size(p):
    """the pad's output size and the keep-aspect-ratio offsets (pad_output_size)"""
    from gstreamer_b200.compositor import pad_output_size
    if p["kar"]:
        return pad_output_size(p["iw"], p["ih"], p["pw"], p["ph"], "keep-aspect-ratio")
    return p["pw"], p["ph"], 0, 0


class Setup:
    """the C-ABI call of a case: destination, pad descriptors, converters (one per distinct conversion)"""

    def __init__(self, lib, mem, case):
        from gstreamer_b200 import _lib
        self.lib, self.case = lib, case
        out, W, H = case["out"], case["W"], case["H"]
        self.di = info(lib, out, W, H, case["dst_odd"])
        if case.get("dst_color"):                                   # the output caps' colorimetry and chroma site
            self.di.color_matrix, self.di.color_range, self.di.chroma_site = case["dst_color"]
        self.dst_ptr, self.dst = mem.upload(np.full(frame_size(out, self.di), 0x5A, dtype=np.uint8))
        n = len(case["pads"])
        self.pads = (_lib.CompPadConvertC * max(n, 1))()
        self.convs, self.frames, self.keep = {}, [], []
        for k, p in enumerate(case["pads"]):
            w, h, xo, yo = output_size(p)
            # a case may bring its own content per pad (comp_fused_cases: worst cases of the pad's conversion)
            a = case["content"](p) if "content" in case else random_frame(lib, p["in_fmt"], p["iw"], p["ih"], p["seed"])
            self.frames.append((a, w, h))
            ii = info(lib, p["in_fmt"], p["iw"], p["ih"], p["odd"])
            tight = unpack(p["in_fmt"], a, info(lib, p["in_fmt"], p["iw"], p["ih"]))
            ptr, handle = mem.upload(pack(p["in_fmt"], tight, ii) if p["odd"] else a)
            self.keep.append(handle)
            conv = None
            if p["in_fmt"] != out or (w, h) != (p["iw"], p["ih"]):
                key = (p["in_fmt"], p["iw"], p["ih"], w, h, str(p["odd"]))
                if key not in self.convs:
                    ci = info(lib, out, w, h)
                    ci.color_matrix, ci.color_range, ci.chroma_site = self.di.color_matrix, self.di.color_range, self.di.chroma_site
                    cfg = _lib.VcsConfigC()
                    lib.b200_vcs_config_init(C.byref(cfg))
                    cfg.method = case.get("method", MITCHELL)
                    hv = C.c_void_p()
                    assert lib.b200_vcs_create(C.byref(ii), C.byref(ci), C.byref(cfg), 0, C.byref(hv)) == 0, key
                    self.convs[key] = hv
                conv = self.convs[key]
            self.pads[k].data, self.pads[k].info, self.pads[k].conv = ptr, ii, conv
            self.pads[k].xpos, self.pads[k].ypos = p["x"] + xo, p["y"] + yo
            self.pads[k].alpha, self.pads[k].op = p["alpha"], p["op"]
        hc = C.c_void_p()
        assert lib.b200_comp_create(FMT[out], W, H, 0, C.byref(hc)) == 0
        self.comp = hc

    def call(self, stream=None):
        return self.lib.b200_comp_blend_convert(self.comp, self.dst_ptr, C.byref(self.di), self.case["bg"], self.pads,
                                                len(self.case["pads"]), stream)

    def routes(self):
        """the route each pad should take: skip, blend, fused or two-pass (what comp.cu's pad_route decides)"""
        from gstreamer_b200 import _lib
        out, W, H = self.case["out"], self.case["W"], self.case["H"]
        r = []
        for k, p in enumerate(self.case["pads"]):
            _, w, h = self.frames[k]
            x, y = self.pads[k].xpos, self.pads[k].ypos
            if out in YUV420:
                x, y = (x + 1) & ~1, (y + 1) & ~1
                dropped = p["alpha"] == 0.0 and p["op"] != 0
            else:
                dropped = int(p["alpha"] * 255) == 0
            visible = x < W and y < H and x + w > 0 and y + h > 0
            conv = self.pads[k].conv
            if dropped or not visible:
                r.append("skip")
            elif not conv:
                r.append("blend")
            else:
                pi = _lib.VcsPlanInfoC()
                assert self.lib.b200_vcs_get_plan_info(conv, C.byref(pi)) == 0
                r.append("fused" if out in YUV420 and pi.kernel_variant == 4 else "two-pass")
        return r

    def close(self):
        for h in self.convs.values():
            self.lib.b200_vcs_destroy(h)
        self.lib.b200_comp_destroy(self.comp)

    def expected(self):
        o = ob.oracle()
        out, W, H = self.case["out"], self.case["W"], self.case["H"]
        n = len(self.case["pads"])
        opads = (ob.OraclePad * max(n, 1))()
        keep = []
        for k, p in enumerate(self.case["pads"]):
            a, w, h = self.frames[k]
            if self.pads[k].conv:
                a = ob.oracle_vcs_convert(ob.vcs_desc(p["iw"], p["ih"], w, h, self.case.get("method", MITCHELL), in_fmt=FMT[p["in_fmt"]],
                                                      out_fmt=FMT[out]), a)
            keep.append(a)
            opads[k].data, opads[k].width, opads[k].height = a.ctypes.data, w, h
            opads[k].stride = 0 if out in YUV420 else w * 4
            opads[k].xpos, opads[k].ypos, opads[k].alpha, opads[k].op = self.pads[k].xpos, self.pads[k].ypos, p["alpha"], p["op"]
        if out in YUV420:
            want = np.zeros(o.oracle_compositor_yuv_size(FMT[out], W, H), dtype=np.uint8)
            assert o.oracle_compositor_yuv(FMT[out], want.ctypes.data, W, H, self.case["bg"], 1, opads, n) == 0
        else:
            want = np.zeros(W * H * 4, dtype=np.uint8)
            o.oracle_compositor(FMT[out], want.ctypes.data, W, H, W * 4, self.case["bg"], opads, n)
        return unpack(out, want, info(self.lib, out, W, H))


def run_case(lib, mem, case, stream, log=None):
    """(output bytes in the default layout, expected bytes, expected routes); `log`: the emulated library, whose launch
    log is checked against the routes"""
    s = Setup(lib, mem, case)
    try:
        routes = s.routes()
        if log is not None:
            check_log(s, routes, route_log(log, case, s))
        assert s.call(stream) == 0
        got = unpack(case["out"], mem.download(s.dst), s.di)
        return got, s.expected(), routes
    finally:
        s.close()


def route_log(emu, case, setup=None):
    """the kernels one call launches (emulated library, record-only)"""
    s = setup or Setup(emu, EmptyMem(), case)
    emu.b200emu_set_record_only(1)
    emu.b200emu_clear_launch_log()
    try:
        assert s.call() == 0
        return [line for line in emu.b200emu_launch_log().decode().split("\n") if line]
    finally:
        emu.b200emu_set_record_only(0)
        if setup is None:
            s.close()


class EmptyMem:
    def upload(self, a):
        a = np.ascontiguousarray(a)
        self.__dict__.setdefault("keep", []).append(a)
        return a.ctypes.data, a


def check_log(s, routes, log):
    """fused pads store through the CompStore kernels and convert nothing into a frame; two-pass converters run their own
    launches once per converter (one batch); blend-kernel runs are comp_*_kernel launches"""
    from gstreamer_b200 import _lib
    fused = [k for k, r in enumerate(routes) if r == "fused"]
    comp_store = [x for x in log if "_comp_kernel" in x]
    assert bool(fused) == bool(comp_store), (routes, log)
    two_pass = {s.pads[k].conv for k, r in enumerate(routes) if r == "two-pass"}
    want = 0
    for h in two_pass:
        pi = _lib.VcsPlanInfoC()
        s.lib.b200_vcs_get_plan_info(h, C.byref(pi))
        want += pi.n_launches_per_convert
    convert = [x for x in log if x.startswith("vcs_") and "_comp_kernel" not in x]
    assert len(convert) == want, (routes, log)
    if not fused and not two_pass:
        assert all(x.startswith("comp_") for x in log), log


def check_bytes(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero(got != want)[0]
        raise AssertionError(f"{what}: {bad.size} bytes differ, first at {bad[0]}: got {got[bad[0]]} want {want[bad[0]]}")


def check_routes(case, routes):
    assert len(routes) == len(case["pads"])
