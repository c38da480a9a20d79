"""TEST INFRASTRUCTURE: worst-case inputs for the scaling kernels, built from each plan's own taps.

A FIR output reaches its extreme only when its window is at full scale on the side of each tap's sign; noise almost never
does that, so the fixed-point arithmetic of a kernel (its tap range, accumulator width, the saturating packs after each
stage) is never driven to its limits by random frames.  This module builds the inputs that do:

  video  Rank-1 XOR frames 255 * (a[x] ^ b[y]) per component, where a and b are the tap-sign patterns of chosen output
         columns and rows (frame borders, tile edges, the interior; windows that do not overlap), each target a maximum
         or a minimum.  Chroma is binary too, so RGB outputs see the matrix's corners (aimed only where chroma planes
         are scaled on their own, see frame()); RGB inputs are patterned per channel.  Seeded random XOR-binary frames reach near-extremes everywhere.
  audio  Full-scale streams whose windows follow the sign of the taps of chosen outputs, found from the resampler's own
         impulse responses (oracle, F64).

plane_model() is a plain float64 statement of the separable 8-bit FIR with the quantised integer taps; the tests use it
to show that each target's pre-clamp value lies beyond the representable range and that the oracle returns the clamped
byte there, i.e. that the content does what it claims.
"""
import ctypes as C
import functools

import numpy as np

import vcs_batch_cases as vb
from oracle import bindings as ob

RGB4 = ("BGRA", "RGBA", "ARGB", "ABGR", "BGRx", "RGBx", "xRGB", "xBGR")
TILE = 16                      # targets at every multiple of this (and one before it): the kernels' tile and warp edges


# ---- taps --------------------------------------------------------------------------------------------------------------
def taps(method, in_size, out_size, precision=6):
    """(n_taps, offset[out], integer taps[out, n]) of one dimension, as the reference's 8-bit scalers quantise them
    (video-scaler.c: 6 bits for 3 and more taps).  1 and 2 taps have no negative weight."""
    o = ob.oracle()
    m, mt, bc = ob.ELEMENT_METHODS[int(method)]
    rs = ob.RS(m, mt, 0, 2.0, 1.0, 0.0, 1 / 3, 1 / 3)
    if bc:
        rs.cubic_b, rs.cubic_c = bc
    off = np.zeros(out_size, dtype=np.uint32)
    t = np.zeros(out_size * 128)
    n = o.oracle_resampler_taps(C.byref(rs), in_size, out_size, off.ctypes.data, t.ctypes.data)
    t = t[: out_size * n].reshape(out_size, n)
    q = np.zeros((out_size, n), dtype=np.int16)
    for i in range(out_size):
        row = np.ascontiguousarray(t[i])
        o.oracle_quantize_taps(row.ctypes.data, q[i].ctypes.data, n, precision)
    return n, off.astype(np.int64), q.astype(np.int64)


def targets(out_size, off, n, extra=()):
    """output indices whose input windows do not overlap: both borders first, then the tile edges, then the interior"""
    cand = [0, out_size - 1, 1, out_size - 2] + list(extra)
    for k in range(TILE, out_size, TILE):
        cand += [k - 1, k]
    cand += [out_size // 2, out_size // 3] + list(range(0, out_size, max(1, n)))
    kept, used = [], np.zeros(int(off.max()) + n + 1, dtype=bool)
    for j in cand:
        if 0 <= j < out_size and j not in kept and not used[off[j]: off[j] + n].any():
            kept.append(j)
            used[off[j]: off[j] + n] = True
    return kept


def pattern(in_size, out_size, method, rng, precision=6):
    """one dimension: (bits a[in_size], {target: inverted}) - inside each target's window a[x] = 1 where its tap is
    negative, flipped for the targets drawn as inverted; random bits elsewhere"""
    n, off, q = taps(method, in_size, out_size, precision)
    a = rng.integers(0, 2, in_size).astype(np.uint8)
    inv = {}
    for j in targets(out_size, off, n):
        inv[j] = int(rng.integers(0, 2))
        a[off[j]: off[j] + n] = (q[j] < 0).astype(np.uint8) ^ inv[j]
    return a, inv


# ---- frame layouts -----------------------------------------------------------------------------------------------------
def components(fmt, w, h):
    """{component: byte index array (rows, cols)} of a frame in the format's default layout, and its byte size"""
    d = ob.vcs_desc(w, h, w, h, 1, in_fmt=ob.FMT[fmt], out_fmt=ob.FMT["BGRA"] if fmt not in RGB4 else ob.FMT["NV12"])
    size = int(ob.vcs_sizes(d)[0])
    s, o = list(d.in_stride), list(d.in_offset)
    cw, ch2 = (w + 1) // 2, (h + 1) // 2

    def grid(off, stride, rows, cols, step=1, first=0):
        return off + np.arange(rows)[:, None] * stride + first + step * np.arange(cols)[None, :]

    if fmt in RGB4:
        return {c: grid(0, 4 * w, h, w, 4, fmt.index(c)) for c in "RGB"} | \
               ({"A": grid(0, 4 * w, h, w, 4, fmt.index("A"))} if "A" in fmt else {}), size
    if fmt in ("NV12", "NV21"):
        u, v = (0, 1) if fmt == "NV12" else (1, 0)
        return {"Y": grid(o[0], s[0], h, w), "U": grid(o[1], s[1], ch2, cw, 2, u), "V": grid(o[1], s[1], ch2, cw, 2, v)}, size
    if fmt in ("I420", "YV12", "Y42B", "Y444"):
        pu, pv = (2, 1) if fmt == "YV12" else (1, 2)
        rows = ch2 if fmt in ("I420", "YV12") else h
        cols = w if fmt == "Y444" else cw
        return {"Y": grid(o[0], s[0], h, w), "U": grid(o[pu], s[pu], rows, cols), "V": grid(o[pv], s[pv], rows, cols)}, size
    pos = {"YUY2": "YUYV", "UYVY": "UYVY", "YVYU": "YVYU"}[fmt]
    y0 = pos.index("Y")
    return {"Y": grid(o[0], s[0], h, w, 2, y0), "U": grid(o[0], s[0], h, cw, 4, pos.index("U")),
            "V": grid(o[0], s[0], h, cw, 4, pos.index("V"))}, size


def subsampled(fmt):
    """(horizontal, vertical) sub-sampling of the chroma components"""
    return {"NV12": (2, 2), "NV21": (2, 2), "I420": (2, 2), "YV12": (2, 2), "Y42B": (2, 1), "YUY2": (2, 1), "UYVY": (2, 1),
            "YVYU": (2, 1)}.get(fmt, (1, 1))


# ---- frames ------------------------------------------------------------------------------------------------------------
def frame(fi, fo, size, method, seed):
    """one worst-case frame of `fi` for the conversion to `fo` at `size`: every component a rank-1 XOR pattern of the
    output's tap signs (its own flips per seed, so that the frames of a batch differ).  Luma and the RGB channels use the
    full-size taps; chroma planes that are scaled on their own (4:2:0 -> the same 4:2:0 family) use the taps at their
    size.  Chroma that is up-sampled into a full-size chain takes the luma pattern at its even pixels: binary, so RGB
    outputs see the matrix's corners, but not aimed at the taps of any one output (the chroma-site-shifted taps of a
    sited chain included); plane_model() confirms the luma targets only."""
    iw, ih, ow, oh = size
    rng = np.random.default_rng(seed)
    idx, nbytes = components(fi, iw, ih)
    out = np.zeros(nbytes, dtype=np.uint8)
    a, _ = pattern(iw, ow, method, rng)
    b, _ = pattern(ih, oh, method, rng)
    sx, sy = subsampled(fi)
    planes = fi in ("NV12", "NV21", "I420", "YV12") and fo in ("NV12", "NV21", "I420", "YV12")
    if planes:
        ac, _ = pattern((iw + 1) // 2, (ow + 1) // 2, method, rng)
        bc, _ = pattern((ih + 1) // 2, (oh + 1) // 2, method, rng)
    for c, ix in idx.items():
        rows, cols = ix.shape
        if c == "A":
            out[ix] = 255
            continue
        if c in "UV" and planes:
            pa, pb = ac[:cols], bc[:rows]
        elif c in "UV":
            pa, pb = a[::sx][:cols], b[::sy][:rows]
        else:
            pa, pb = a, b
        flip = int(rng.integers(0, 2))
        out[ix] = 255 * (1 ^ flip ^ pa[None, :] ^ pb[:, None])
    return out


# batch rows of the knobs that select a kernel form no batch row reaches: the 2:1 kernel's plain tap tables
KNOB_ROWS = [vb.Row("nv12-bgra-2to1-plain", "NV12", "BGRA", (256, 144, 128, 72), 3, "vcs_lanczos2_kernel",
                    ("vcs_lanczos2_kernel<true, 4, 60, 1, false>",), site=2, knob="B200_L2_X4=0")]


class WorstHandle(vb.Handle):
    """a batch row's handle (tests/vcs_batch_cases.py) whose frames are worst cases: even seeds aimed at the row's own
    taps, odd seeds random XOR-binary, so every frame of a batch is a different extreme"""

    def frame(self, seed):
        r = self.row
        f = frame(r.fi, r.fo, r.size, r.method, seed) if seed % 2 == 0 else random_binary(r.fi, r.size, seed)
        assert f.size == self.in_size
        return f


def random_binary(fi, size, seed):
    """seeded XOR-binary frame: every component 255 * (a[x] ^ b[y]) with random bit vectors a, b"""
    iw, ih = size[:2]
    rng = np.random.default_rng(seed)
    idx, nbytes = components(fi, iw, ih)
    out = np.zeros(nbytes, dtype=np.uint8)
    for c, ix in idx.items():
        rows, cols = ix.shape
        a, b = rng.integers(0, 2, cols), rng.integers(0, 2, rows)
        out[ix] = 255 if c == "A" else 255 * (a[None, :] ^ b[:, None])
    return out


# ---- the float64 model ---------------------------------------------------------------------------------------------------
def plane_model(plane, method, out_w, out_h):
    """the separable 8-bit FIR of one plane in float64 with the integer taps, in gst_video_scaler_2d's pass order
    (horizontal first unless the last output row's window starts below row out_h): first pass, round, clamp, second
    pass, round, clamp.  Returns (ideal, staged, targets): ideal is the un-clamped 2-D value sum(h * v * p) / 64^2,
    staged the byte each stage's saturating pack gives, targets the (rows, columns) pattern() aimed at.  Only for 3 and
    more taps in both dimensions (the n-tap scalers)."""
    p = plane.astype(np.float64)
    nh, oh_, qh = taps(method, p.shape[1], out_w)
    nv, ov, qv = taps(method, p.shape[0], out_h)
    assert nh >= 3 and nv >= 3
    H = np.zeros((out_w, p.shape[1]))
    for j in range(out_w):
        H[j, oh_[j]: oh_[j] + nh] = qh[j] / 64.0
    V = np.zeros((out_h, p.shape[0]))
    for i in range(out_h):
        V[i, ov[i]: ov[i] + nv] = qv[i] / 64.0
    ideal = V @ p @ H.T
    if ov[-1] <= out_h:
        staged = np.clip(np.floor(V @ np.clip(np.floor(p @ H.T + 0.5), 0, 255) + 0.5), 0, 255)
    else:
        staged = np.clip(np.floor(np.clip(np.floor(V @ p + 0.5), 0, 255) @ H.T + 0.5), 0, 255)
    return ideal, staged, (targets(out_h, ov, nv), targets(out_w, oh_, nh))


# ---- audio -------------------------------------------------------------------------------------------------------------
FULL_SCALE = {"S16": 32767, "S32": 2147483647, "F32": 1.0, "F64": 1.0}


@functools.lru_cache(maxsize=None)
def ars_response(a, b, q, n_in):
    """W[k, m]: output k of a fresh mono F64 stream of n_in frames for a unit impulse at input m (the oracle's resampler,
    default options) - each row is the window and the taps that output uses"""
    o = ob.oracle()
    ofmt = ob.AUDIO_FORMATS["F64"][0]
    cols = []
    for m in range(n_in):
        h = o.oracle_ars_new_fmt(a, b, 1, q, ofmt)
        x = np.zeros(n_in)
        x[m] = 1.0
        cap = int(n_in * b / a) + 64
        y = np.zeros(cap)
        n = o.oracle_ars_process_any(h, x.ctypes.data, n_in, y.ctypes.data, cap)
        o.oracle_ars_free(h)
        cols.append(y[:n])
    return np.stack(cols, axis=1)


def ars_stream(a, b, q, n, channels, seed):
    """(x[n, channels] of +-1, {channel: [(output, +1 max / -1 min)]}, the smallest sum of |taps| of a target window, whether the filter is periodic) for a fresh stream a -> b at quality q: per
    channel, outputs whose windows do not overlap are driven to their maximum or minimum (x = +-1 on the sign of each
    tap); every other sample is a random +-1.  The windows come from ars_response(); where the filter has one row per
    phase (FULL mode) they repeat every in_step input frames and out_step outputs, so targets cover the whole stream."""
    o = ob.oracle()
    h = o.oracle_ars_new_fmt(a, b, 1, q, ob.AUDIO_FORMATS["F64"][0])
    info = [C.c_int() for _ in range(6)]
    o.oracle_ars_info(h, *[C.byref(v) for v in info])
    o.oracle_ars_free(h)
    n_taps, n_phases, in_step, out_step, full = (v.value for v in info[:5])
    W = ars_response(a, b, q, min(n, 2 * n_taps + 3 * in_step, 1500))
    period = (in_step, out_step) if full and n_phases == out_step else None
    rows = []
    for k in range(W.shape[0]):
        nz = np.flatnonzero(W[k])
        # whole windows only, clear of the start, and whose extreme lies beyond full scale
        if nz.size and nz[-1] - nz[0] + 1 == n_taps and nz[0] > 0 and np.abs(W[k]).sum() > 1.01:
            rows.append((k, nz[0], np.where(W[k, nz[0]: nz[-1] + 1] < 0, -1.0, 1.0)))
    l1 = min(np.abs(W[k]).sum() for k, _, _ in rows)
    rng = np.random.default_rng(seed)
    x = rng.choice([-1.0, 1.0], size=(n, channels))
    aims = {}
    for c in range(channels):
        used = np.zeros(n, dtype=bool)
        aims[c] = []
        for s in range(0, (n // period[0] + 1) if period else 1):
            for k, start, sign in rows:
                k1, m = (k + s * period[1], start + s * period[0]) if period else (k, start)
                if m + n_taps > n or used[m: m + n_taps].any():
                    continue
                d = 1 if rng.integers(0, 2) else -1
                x[m: m + n_taps, c] = d * sign
                used[m: m + n_taps] = True
                aims[c].append((k1, d))
    return x, aims, l1, bool(period)


def run_ars_case(transform, fmt, cfg, scale, seed, n_total=9000):
    """the worst-case stream of `cfg` in buffers of uneven length, then a silent drain, through `transform(x, n, cap)`
    (the product) and the oracle; every buffer byte-identical.  Returns the saturated targets the oracle showed."""
    a, b, ch, q = cfg
    ofmt, _, dt, _ = ob.AUDIO_FORMATS[fmt]
    x, aims, _, full = ars_stream(a, b, q, n_total, ch, seed)
    xs = to_format(x, fmt, scale)
    o = ob.oracle()
    ho = o.oracle_ars_new_fmt(a, b, ch, q, ofmt)
    outs = []
    try:
        pos = 0
        for n in (n_total * 8 // 15, 7, n_total // 3, n_total, None):     # the last buffer takes what is left
            chunk = None
            if n is None:
                n = o.oracle_ars_max_latency(ho)
            else:
                chunk = np.ascontiguousarray(xs[pos: pos + n])
                n = chunk.shape[0]
                pos += n
            cap = int(n * b / a) + 64
            want = np.zeros((cap, ch), dtype=dt)
            nw = o.oracle_ars_process_any(ho, chunk.ctypes.data if chunk is not None else None, n, want.ctypes.data, cap)
            ng, got = transform(chunk, n, cap)
            assert ng == nw and got[:ng].tobytes() == want[:nw].tobytes(), (fmt, cfg, n)
            outs.append(want[:nw])
    finally:
        o.oracle_ars_free(ho)
    return np.concatenate(outs), aims, full


def ars_scale(fmt, cfg):
    """full scale for the float formats (outputs beyond +-1 must come through unclamped); for the integer formats the
    level at which the weakest target window sums to 1.1x full scale, so that it saturates without the reference's
    accumulators wrapping (full scale itself wraps them; the device must then wrap alike - run_ars_case at scale 1)"""
    if fmt in ("F32", "F64"):
        return 1.0
    a, b, ch, q = cfg
    return min(1.0, 1.1 / ars_stream(a, b, q, 4000, 1, 0)[2])


def check_saturation(y, aims, fmt):
    """the oracle's output at every target: the format's extreme for the integer formats (the window's exact sum lies
    beyond it), beyond full scale and unclamped for the float formats"""
    hits = 0
    for c, lst in aims.items():
        for k, d in lst:
            if k >= y.shape[0]:
                continue
            v = y[k, c]
            if fmt in ("S16", "S32"):
                dt = ob.AUDIO_FORMATS[fmt][2]
                assert v == (np.iinfo(dt).max if d > 0 else np.iinfo(dt).min), (fmt, c, k, d, v)
            else:
                assert v * d > 1.0, (fmt, c, k, d, v)
            hits += 1
    return hits


def to_format(x, fmt, scale=1.0):
    """+-1 samples in the sample format at `scale` of full scale: at 1, the integer formats' extremes"""
    dt = ob.AUDIO_FORMATS[fmt][2]
    if fmt in ("S16", "S32"):
        if scale == 1.0:
            return np.where(x > 0, np.iinfo(dt).max, np.iinfo(dt).min).astype(dt)
        return np.round(x * scale * np.iinfo(dt).max).astype(dt)
    return (x * scale).astype(dt)
