"""TEST INFRASTRUCTURE: the compositor's pixel arithmetic over its whole input domain.

The kernels (comp.cu) reach their bytes by arithmetic that is exact only by narrow arguments: div255 on two 16-bit lanes
per register, a reciprocal table for the overlay division, saturating packs whose selectors depend on where the alpha
byte sits, the wrapping 32-bit statement of the 10 / 12 / 16-bit blends.  This module holds

  model     plain integer statements of every pixel operation (floor division, no tricks), written once for numpy and
            torch int64 arrays, so that the device's expected bytes can be computed on the device;
  domains   frames that carry a whole input domain through one call: pad 0 is SOURCE at alpha 1.0 and copies an
            arbitrary destination (alpha byte included), then up to 63 operator pads, each over its own band of rows
            with its own pad alpha, apply the operator under test;
  alphas    the pad alphas that reach each integer alpha, and the edges where the quantisation changes.

It never calls the oracle: tests/test_comp_domain.py pins the model against the oracle and the reference build.
"""
import ctypes as C

import numpy as np

RGB = {"RGBA": (11, 3), "BGRA": (12, 3), "ARGB": (13, 0), "ABGR": (14, 0)}     # format, byte index of alpha
# 4:4:4 planar outputs of every depth: (format, significant bits)
YUV = {"Y444": (20, 8), "Y444_10LE": (47, 10), "Y444_12LE": (77, 12), "Y444_16LE": (88, 16)}
SOURCE, OVER, ADD = 0, 1, 2
CHECKER, BLACK, WHITE, TRANSPARENT = 0, 1, 2, 3
MAX_PADS = 64
COPY = 1 << 16                 # the integer alpha of a pad that is copied, not blended (above every blend alpha)


def _where(c, a, b):
    if isinstance(c, np.ndarray):
        return np.where(c, a, b)
    import torch
    return torch.where(c, a, b)


# ---- model ---------------------------------------------------------------------------------------------------------------
def rgb_alpha(alpha):
    """the integer pad alpha of a packed RGB pad: CLAMP ((gint) (alpha * 255), 0, 255); 0 drops the pad"""
    return min(max(int(alpha * 255), 0), 255)


def yuv_alpha(alpha, op, nbits):
    """the integer pad alpha of a planar pad: COPY for alpha 1.0 and SOURCE, 0 (dropped) for alpha 0, else
    CLAMP ((gint) (alpha * (2^n - 1)), 0, 2^n - 1)"""
    if op == SOURCE or alpha == 1.0:
        return COPY
    rng = (1 << nbits) - 1
    return min(max(int(alpha * rng), 0), rng)


def mul_alpha(as_, k):
    """the source alpha byte under pad alpha k: floor(as * k / 255)"""
    return as_ * k // 255


def blend(s, d, a):
    """OVER / ADD on an opaque background, one colour byte: floor((s*a + d*(255-a)) / 255)"""
    return (s * a + d * (255 - a)) // 255


def overlay(s, d, a, da):
    """OVER on a transparent background, one colour byte: ad = floor(da*(255-a)/255), floor((s*a + d*ad) / (a+ad))
    capped at 255, 255 when a + ad = 0"""
    ad = da * (255 - a) // 255
    asum = a + ad
    q = (s * a + d * ad) // _where(asum == 0, 1, asum)
    return _where(asum == 0, 255, q.clip(max=255))


def overlay_alpha(a, da, add):
    """the alpha byte OVER (a + ad) or ADD ((da + a) mod 256) leaves on a transparent background"""
    return (da + a) % 256 if add else a + da * (255 - a) // 255


def blend_u8(s, d, a):
    """an 8-bit plane sample: floor((d*(256-a) + s*a) / 256)"""
    return (d * (256 - a) + s * a) // 256


def blend_wide_unclamped(s, d, a, nbits):
    """a 10 / 12 / 16-bit plane sample, as the wrapping 32-bit statement computes it before its clamp:
    (((d << n) + (s - d) * a) mod 2^32) >> n, with samples anywhere in the 16-bit range"""
    return (((d << nbits) + (s - d) * a) % (1 << 32)) >> nbits


def blend_wide(s, d, a, nbits):
    """the same, then the signed-to-unsigned 16-bit clamp"""
    return blend_wide_unclamped(s, d, a, nbits).clip(0, 65535)


def _i64(a):
    return a.astype(np.int64) if isinstance(a, np.ndarray) else a.long()


def _like(a, ref):
    return a.astype(ref.dtype) if isinstance(a, np.ndarray) else a.to(ref.dtype)


def _copy(a):
    return a.copy() if isinstance(a, np.ndarray) else a.clone()


def rgb_expected(fmt, bg, d, s, bands):
    """the model's output of a domain call (rgb_pads): d[H, W, 4] copied, then each band (y0, y1, alpha, op) of s
    applied to rows y0 .. y1 - 1"""
    ai = RGB[fmt][1]
    out = _copy(d)
    for y0, y1, alpha, op in bands:
        k = rgb_alpha(alpha)
        if k == 0:
            continue
        if op == SOURCE and k == 255:
            out[y0:y1] = s[y0:y1]
            continue
        sc, dc = _i64(s[y0:y1]), _i64(out[y0:y1])
        a = mul_alpha(sc[..., ai], k)
        res = _copy(sc if op == SOURCE else dc)
        if op == SOURCE:
            res[..., ai] = a
        elif bg != TRANSPARENT:
            for c in range(4):
                res[..., c] = 255 if c == ai else blend(sc[..., c], dc[..., c], a)
        else:
            da = dc[..., ai]
            for c in range(4):
                res[..., c] = overlay_alpha(a, da, op == ADD) if c == ai else overlay(sc[..., c], dc[..., c], a, da)
        out[y0:y1] = _like(res, out)
    return out


def yuv_expected(nbits, d, s, bands):
    """the model's output of a domain call (yuv_pads) on samples d[3, H, W] / s (uint8, or int32 holding 16-bit samples)"""
    out = _copy(d)
    for y0, y1, alpha, op in bands:
        a = yuv_alpha(alpha, op, nbits)
        if a == 0:
            continue
        if a == COPY:
            out[:, y0:y1] = s[:, y0:y1]
            continue
        sc, dc = _i64(s[:, y0:y1]), _i64(out[:, y0:y1])
        out[:, y0:y1] = _like(blend_u8(sc, dc, a) if nbits == 8 else blend_wide(sc, dc, a, nbits), out)
    return out


# ---- alphas --------------------------------------------------------------------------------------------------------------
def alpha_for(k, rng):
    """a pad alpha whose quantisation at `rng` (255, 1023, 4095, 65535) is the integer k"""
    return (k + 0.5) / rng


def alpha_edges(rng, ks=None):
    """k / rng and both of its floating-point neighbours, for every k (or the given ones): where the quantisation steps"""
    out = []
    for k in (range(rng + 1) if ks is None else ks):
        v = k / rng
        out += [float(np.nextafter(v, -1.0)), v, float(np.nextafter(v, 2.0))]
    return [a for a in out if a >= 0.0]


# ---- domains -------------------------------------------------------------------------------------------------------------
def pair_grid(n, bits=8):
    """(s, d) for pair index 0 .. n - 1 over all 2^bits x 2^bits pairs (int64 numpy arrays)"""
    q = np.arange(n, dtype=np.int64) % (1 << (2 * bits))
    return q & ((1 << bits) - 1), q >> bits


def bands_of(alphas, rows, op, first=0):
    """one band of `rows` rows per pad alpha, from row `first` on: [(y0, y1, alpha, op)]"""
    return [(first + i * rows, first + (i + 1) * rows, a, op) for i, a in enumerate(alphas)]


def chunks(seq, n):
    return [seq[i: i + n] for i in range(0, len(seq), n)]


class Host:
    """numpy frames at host addresses: the emulated library (its 'device memory' is host memory)"""
    xp = np

    def __init__(self, lib):
        self.lib = lib

    @staticmethod
    def ptr(a):
        return a.ctypes.data

    def sync(self):
        pass

    @staticmethod
    def asarray(a):
        return np.ascontiguousarray(a)

    @staticmethod
    def to_numpy(a):
        return a


class Device:
    """torch tensors on cuda:0: the product's library"""

    def __init__(self):
        import torch
        from gstreamer_b200._lib import lib
        self.lib, self.torch, self.xp = lib, torch, torch

    @staticmethod
    def ptr(a):
        return a.data_ptr()

    def sync(self):
        self.torch.cuda.synchronize()

    def asarray(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).cuda() if isinstance(a, np.ndarray) else a.contiguous()

    @staticmethod
    def to_numpy(a):
        return a.cpu().numpy()


def _pad_struct():
    from gstreamer_b200 import _lib
    return _lib


def rgb_pads(mem, fmt, bg, d, s, bands, dst=None, dst_stride=None, entry="blend"):
    """one b200_comp_blend call (entry "blend"; "convert": b200_comp_blend_convert, no converters) over d, s [H, W, 4]
    (arrays of `mem`): pad 0 SOURCE at 1.0 copies d, then one pad per band of s.  Returns the destination (a fresh
    array, or `dst` written at `dst_stride` bytes per row)."""
    _lib = _pad_struct()
    H, W = int(d.shape[0]), int(d.shape[1])
    fmt_id = RGB[fmt][0]
    n = 1 + len(bands)
    rects = [(mem.ptr(d), 0, H, 1.0, SOURCE)] + [(mem.ptr(s) + y0 * W * 4, y0, y1 - y0, a, op) for y0, y1, a, op in bands]
    pads = ((_lib.CompPadC if entry == "blend" else _lib.CompPadConvertC) * n)()
    for p, (ptr, y, h, alpha, op) in zip(pads, rects):
        if entry == "blend":
            p.data, p.width, p.height, p.stride = ptr, W, h, W * 4
        else:
            p.data, p.info, p.conv = ptr, yuv_info(mem.lib, fmt_id, W, h), None
        p.xpos, p.ypos, p.alpha, p.op = 0, y, alpha, op
    if dst is None:
        dst, dst_stride = (np.zeros((H, W, 4), np.uint8) if mem.xp is np else mem.torch.empty_like(d)), W * 4
    h = C.c_void_p()
    assert mem.lib.b200_comp_create(fmt_id, W, H, 0, C.byref(h)) == 0
    try:
        if entry == "blend":
            st = mem.lib.b200_comp_blend(h, mem.ptr(dst), dst_stride, bg, pads, n, None)
        else:
            di = yuv_info(mem.lib, fmt_id, W, H)
            di.stride[0] = dst_stride
            st = mem.lib.b200_comp_blend_convert(h, mem.ptr(dst), C.byref(di), bg, pads, n, None)
        assert st == 0, st
        mem.sync()
    finally:
        mem.lib.b200_comp_destroy(h)
    return dst


def yuv_info(lib, fmt, w, h):
    """the default layout of a w x h frame of `fmt`"""
    _lib = _pad_struct()
    i = _lib.VideoInfoC()
    assert lib.b200_video_info_set_format(C.byref(i), fmt, w, h) == 0
    return i


def yuv_planes_to_bytes(a, nbits):
    """samples [3, H, W] -> the frame's bytes (planes back to back, little-endian 16-bit samples above 8 bits)"""
    if nbits == 8:
        return a
    if isinstance(a, np.ndarray):
        return np.ascontiguousarray(a.astype("<u2")).view(np.uint8)
    import torch
    return a.to(torch.int32).to(torch.int16).contiguous().view(torch.uint8)


def yuv_bytes_to_planes(b, nbits, shape):
    if nbits == 8:
        return b.reshape(shape)
    if isinstance(b, np.ndarray):
        return b.view("<u2").reshape(shape).astype(np.int32)
    import torch
    return (b.view(torch.int16).to(torch.int32) & 0xffff).reshape(shape)


def yuv_pads(mem, name, d, s, bands, entry="yuv"):
    """one b200_comp_blend_yuv (entry "yuv") or b200_comp_blend_convert (entry "convert", no converters) call on a 4:4:4
    output of `name`: samples d, s [3, H, W] (uint8, or int32 holding 16-bit samples); pad 0 SOURCE at 1.0 copies d, then
    one pad per band of s.  Returns the output's samples."""
    _lib = _pad_struct()
    fmt, nbits = YUV[name]
    H, W = int(d.shape[1]), int(d.shape[2])
    lib = mem.lib
    frames = [yuv_planes_to_bytes(d, nbits).reshape(-1)]
    infos = [yuv_info(lib, fmt, W, H)]
    for y0, y1, _, _ in bands:
        frames.append(yuv_planes_to_bytes(s[:, y0:y1], nbits).reshape(-1))
        infos.append(yuv_info(lib, fmt, W, y1 - y0))
    frames = [mem.asarray(f) for f in frames]
    n = len(frames)
    Pad = _lib.CompPadYuvC if entry == "yuv" else _lib.CompPadConvertC
    pads = (Pad * n)()
    for i, (f, info) in enumerate(zip(frames, infos)):
        pads[i].data, pads[i].info = mem.ptr(f), info
        if entry != "yuv":
            pads[i].conv = None
        if i == 0:
            pads[i].xpos, pads[i].ypos, pads[i].alpha, pads[i].op = 0, 0, 1.0, SOURCE
        else:
            y0, _, alpha, op = bands[i - 1]
            pads[i].xpos, pads[i].ypos, pads[i].alpha, pads[i].op = 0, y0, alpha, op
    di = yuv_info(lib, fmt, W, H)
    out = mem.asarray(np.zeros(W * H * 3 * (1 if nbits == 8 else 2), np.uint8))
    h = C.c_void_p()
    assert lib.b200_comp_create(fmt, W, H, 0, C.byref(h)) == 0
    try:
        fn = lib.b200_comp_blend_yuv if entry == "yuv" else lib.b200_comp_blend_convert
        st = fn(h, mem.ptr(out), C.byref(di), BLACK, pads, n, None)
        assert st == 0, st
        mem.sync()
    finally:
        lib.b200_comp_destroy(h)
    return yuv_bytes_to_planes(out, nbits, (3, H, W))


# ---- launch chunks: many pads at arbitrary rectangles -----------------------------------------------------------------------
def random_pads(rng, W, H, n, planes=None, nbits=8):
    """n pads of random size and position (clipping every edge, negative and odd coordinates), alpha and operator:
    [(frame, x, y, alpha, op)], frame [h, w, 4] uint8 (planes=None) or [3, h, w] samples"""
    alphas = (0.0, 0.003, alpha_for(1, 255), 0.3, 0.5, alpha_for(254, 255), 0.999, 1.0, 1.2)
    pads = []
    for _ in range(n):
        w, h = int(rng.integers(1, W + 9)), int(rng.integers(1, H + 9))
        x, y = int(rng.integers(-w + 1, W)), int(rng.integers(-h + 1, H))
        if planes is None:
            f = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        else:
            f = rng.integers(0, 1 << nbits, (3, h, w)).astype(np.uint8 if nbits == 8 else np.int32)
        pads.append((f, x, y, float(rng.choice(alphas)), int(rng.integers(0, 3))))
    return pads


def _clip(W, H, f, x, y, hw):
    h, w = hw
    x0, y0, x1, y1 = max(x, 0), max(y, 0), min(x + w, W), min(y + h, H)
    return (x0, y0, x1, y1) if x1 > x0 and y1 > y0 else None


def rgb_expected_pads(fmt, bg, d, pads):
    """the model's output of rgb_pads_call: d [H, W, 4] copied, then every pad over its clipped rectangle"""
    H, W = d.shape[:2]
    out = _copy(d)
    for f, x, y, alpha, op in pads:
        r = _clip(W, H, f, x, y, f.shape[:2])
        if r is None:
            continue
        x0, y0, x1, y1 = r
        # the pad over the destination rows it covers, as a one-band call of the same operator
        sub = out[y0:y1, x0:x1]
        src = f[y0 - y: y1 - y, x0 - x: x1 - x]
        out[y0:y1, x0:x1] = rgb_expected(fmt, bg, sub, src, [(0, y1 - y0, alpha, op)])
    return out


def yuv_expected_pads(nbits, d, pads):
    """the same for 4:4:4 planes [3, H, W]"""
    H, W = d.shape[1:]
    out = _copy(d)
    for f, x, y, alpha, op in pads:
        r = _clip(W, H, f, x, y, f.shape[1:])
        if r is None:
            continue
        x0, y0, x1, y1 = r
        out[:, y0:y1, x0:x1] = yuv_expected(nbits, out[:, y0:y1, x0:x1], f[:, y0 - y: y1 - y, x0 - x: x1 - x],
                                            [(0, y1 - y0, alpha, op)])
    return out


def rgb_pads_call(mem, fmt, bg, d, pads, entry="blend", dst_offset=4, row_pad=4, fill=0x5A):
    """pad 0 (SOURCE at 1.0) copies d [H, W, 4], then `pads` (random_pads) through b200_comp_blend (entry "blend"),
    b200_comp_blend_convert ("convert") or b200_comp_blend_host ("host", host memory), into a destination that starts
    `dst_offset` bytes into its allocation with `row_pad` bytes after each row.  Returns (status, allocation bytes, the
    frame [H, W, 4] inside it)."""
    _lib = _pad_struct()
    H, W = d.shape[:2]
    stride = W * 4 + row_pad
    frames = [mem.asarray(d)] + [mem.asarray(f) for f, *_ in pads]
    rects = [(0, 0, 1.0, SOURCE)] + [(x, y, a, op) for _, x, y, a, op in pads]
    n = len(frames)
    pads_c = ((_lib.CompPadConvertC if entry == "convert" else _lib.CompPadC) * n)()
    for p, fr, (x, y, alpha, op) in zip(pads_c, frames, rects):
        h, w = int(fr.shape[0]), int(fr.shape[1])
        if entry == "convert":
            p.data, p.info, p.conv = mem.ptr(fr), yuv_info(mem.lib, RGB[fmt][0], w, h), None
        else:
            p.data, p.width, p.height, p.stride = mem.ptr(fr), w, h, w * 4
        p.xpos, p.ypos, p.alpha, p.op = x, y, alpha, op
    buf = mem.asarray(np.full(dst_offset + stride * H, fill, np.uint8))
    h = C.c_void_p()
    assert mem.lib.b200_comp_create(RGB[fmt][0], W, H, 0, C.byref(h)) == 0
    try:
        if entry == "blend":
            st = mem.lib.b200_comp_blend(h, mem.ptr(buf) + dst_offset, stride, bg, pads_c, n, None)
        else:
            di = yuv_info(mem.lib, RGB[fmt][0], W, H)
            di.stride[0] = stride
            st = mem.lib.b200_comp_blend_convert(h, mem.ptr(buf) + dst_offset, C.byref(di), bg, pads_c, n, None)
        mem.sync()
    finally:
        mem.lib.b200_comp_destroy(h)
    b = mem.to_numpy(buf)
    return st, b, b[dst_offset:].reshape(H, stride)[:, : W * 4].reshape(H, W, 4)


def yuv_pads_call(mem, name, d, pads, entry="yuv", fill=0x5A):
    """the same for a 4:4:4 output of `name` through b200_comp_blend_yuv or b200_comp_blend_convert; the destination's
    rows carry 4 bytes of padding.  Returns (status, allocation bytes, samples [3, H, W])."""
    _lib = _pad_struct()
    fmt, nbits = YUV[name]
    es = 1 if nbits == 8 else 2
    H, W = d.shape[1:]
    frames = [d] + [f for f, *_ in pads]
    rects = [(0, 0, 1.0, SOURCE)] + [(x, y, a, op) for _, x, y, a, op in pads]
    Pad = _lib.CompPadYuvC if entry == "yuv" else _lib.CompPadConvertC
    pads_c = (Pad * len(frames))()
    keep = []
    for p, fr, (x, y, alpha, op) in zip(pads_c, frames, rects):
        keep.append(mem.asarray(yuv_planes_to_bytes(np.ascontiguousarray(fr), nbits).reshape(-1)))
        h, w = int(fr.shape[1]), int(fr.shape[2])
        info = yuv_info(mem.lib, fmt, w, h)
        for k in range(3):                                         # planes back to back, rows without padding
            info.stride[k], info.offset[k] = w * es, k * w * es * h
        p.data, p.info = mem.ptr(keep[-1]), info
        if entry != "yuv":
            p.conv = None
        p.xpos, p.ypos, p.alpha, p.op = x, y, alpha, op
    di = yuv_info(mem.lib, fmt, W, H)
    stride = W * es + 4
    for k in range(3):
        di.stride[k], di.offset[k] = stride, k * stride * H
    buf = mem.asarray(np.full(3 * stride * H, fill, np.uint8))
    h = C.c_void_p()
    assert mem.lib.b200_comp_create(fmt, W, H, 0, C.byref(h)) == 0
    try:
        fn = mem.lib.b200_comp_blend_yuv if entry == "yuv" else mem.lib.b200_comp_blend_convert
        st = fn(h, mem.ptr(buf), C.byref(di), BLACK, pads_c, len(frames), None)
        mem.sync()
    finally:
        mem.lib.b200_comp_destroy(h)
    b = mem.to_numpy(buf)
    planes = b.reshape(3, H, stride)[:, :, : W * es].reshape(-1)
    return st, b, yuv_bytes_to_planes(np.ascontiguousarray(planes), nbits, (3, H, W))
