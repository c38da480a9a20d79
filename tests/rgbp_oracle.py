"""TEST INFRASTRUCTURE: expected bytes of the planar RGB outputs (RGBP / BGRP) from the CPU oracle.

The reference unpacks and packs RGBP / BGRP through ARGB (video-format.c:7478, PACK_RGBP; pack_RGBP / pack_BGRP
:7496-7536 store the R, G and B bytes of each ARGB pixel in their own planes and drop the alpha), so its chain is the
packed RGB one.  The expected frame is therefore the oracle's packed frame of the same conversion, de-interleaved:
  - YUV inputs: the oracle's BGRx frame.  One exception: I420 / YV12 at an unchanged size, where BGRx takes the
    convert_I420_BGRA table row (nearest chroma) and planar RGB has no such row (video-converter.c:8766-8806) and runs
    the chain.  Unpacking I420 and NV12 gives the same AYUV lines, so that case is the oracle's chain on the same
    frame repacked as NV12.
  - packed RGB inputs: the oracle's conversion to another packed byte order (the matrix-free chain, not the same-format
    table row), whose padding / alpha byte is dropped.
Borders (add-borders rectangle) come out of the packed frame too: border_argb's R, G, B bytes per plane.
"""
import ctypes as C

import numpy as np

from oracle import bindings as ob

FMT = dict(ob.FMT, RGBP=99, BGRP=100)
RGB = ("BGRA", "RGBA", "ARGB", "ABGR", "BGRx", "RGBx", "xRGB", "xBGR")
_BYTES = {"BGRx": (2, 1, 0), "RGBx": (0, 1, 2)}     # memory byte of R, G, B in the packed frame


def default_layout(ow, oh):
    """video-info.c:1030-1041 (the Y444 case): three planes of stride ROUND_UP_4 (w)"""
    s = (ow + 3) & ~3
    return [s, s, s], [0, s * oh, 2 * s * oh]


def frame_size(layout, oh):
    return max(layout[1][k] + layout[0][k] * oh for k in range(3))


def _as_nv12(fi, iw, ih, frame):
    """an I420 / YV12 frame (default layout) repacked as NV12 (default layout)"""
    src = ob.vcs_desc(iw, ih, iw, ih, 1, in_fmt=FMT[fi], out_fmt=8)
    dst = ob.vcs_desc(iw, ih, iw, ih, 1, in_fmt=FMT["NV12"], out_fmt=8)
    nv = np.zeros(ob.vcs_sizes(dst)[0], dtype=np.uint8)
    sy, dy = src.in_stride[0], dst.in_stride[0]
    for y in range(ih):
        nv[dst.in_offset[0] + y * dy: dst.in_offset[0] + y * dy + iw] = frame[src.in_offset[0] + y * sy: src.in_offset[0] + y * sy + iw]
    pu, pv = (1, 2) if fi == "I420" else (2, 1)
    cw, ch = (iw + 1) // 2, (ih + 1) // 2
    for y in range(ch):
        row = nv[dst.in_offset[1] + y * dst.in_stride[1]:]
        row[0: 2 * cw: 2] = frame[src.in_offset[pu] + y * src.in_stride[pu]:][:cw]
        row[1: 2 * cw: 2] = frame[src.in_offset[pv] + y * src.in_stride[pv]:][:cw]
    return nv


def oracle_rgbp(fi, fo, size, method, frame, site=None, matrix=None, rng=None, layout=None, dest=None,
                border=0xff000000, fill=0x5A):
    """the whole RGBP / BGRP output frame (planes at `layout` = (strides, offsets), other bytes = fill)"""
    iw, ih, ow, oh = size
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    po = "RGBx" if fi == "BGRx" else "BGRx"
    rw, rh = ow, oh                                   # the size the chain scales to (the rectangle with add-borders)
    if dest:
        rw, rh = min(dest[2], ow - dest[0]), min(dest[3], oh - dest[1])
    if fi in ("I420", "YV12") and (rw, rh) == (iw, ih):
        frame, fi = _as_nv12(fi, iw, ih, frame), "NV12"
    d = ob.vcs_desc(iw, ih, ow, oh, method, in_fmt=FMT[fi], out_fmt=FMT[po], site=site, matrix=matrix, rng=rng)
    if dest:
        packed = ob.oracle_vcs_convert_dest(d, frame, dest, border)
    else:
        packed = np.zeros(ob.vcs_sizes(d)[1], dtype=np.uint8)
        assert ob.oracle().oracle_vcs_convert(C.byref(d), frame.ctypes.data, packed.ctypes.data) == 0
    packed = packed.reshape(oh, ow, 4)
    layout = layout or default_layout(ow, oh)
    out = np.full(frame_size(layout, oh), fill, dtype=np.uint8)
    rgb = _BYTES[po]
    comps = (rgb[2], rgb[1], rgb[0]) if fo == "BGRP" else rgb    # plane k's byte in the packed pixel
    for k in range(3):
        st, off = layout[0][k], layout[1][k]
        out[off: off + st * oh].reshape(oh, st)[:, :ow] = packed[:, :, comps[k]]
    return out
