#!/usr/bin/env python
"""tests/golden/make_comp_convert.py — compositor convert pads from the REFERENCE build (oracle/_ref): each converted pad
through the option-less GstVideoConverter a GstVideoAggregatorConvertPad creates (refdrv_video, method -1) from the pad's
caps to the output's format, colour matrix, range and chroma site at the pad's output size, then the reference blend
(refdrv_comp).  Writes comp_convert.npz / comp_convert_cases.json, read by tests/test_golden_comp_convert.py.
Some outputs carry a colorimetry other than their size's default (BT709, full range on a small frame), so that a pad
converts to the output's colorimetry and not to the one its own size would give.  A pad whose reference conversion differs
from the oracle restatement's (some chroma bytes of small frames on the 4:2:0 family change and into packed RGB, a
converter matter that the converter's own tests track) is drawn again, so that every difference this fixture can show
belongs to the compositor."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import bindings as ob  # noqa: E402
import comp_convert_cases as cc  # noqa: E402


def main():
    from gstreamer_b200._lib import lib                          # the default layouts and colorimetry (b200_video_info)
    o, r = ob.oracle(), ob.ref()
    rng = np.random.default_rng(2718)
    arrays, cases = {}, []
    outs = ["NV12", "I420", "YV12", "NV21", "BGRA", "RGBA", "ARGB", "ABGR"]
    for t in range(16):
        out = outs[t % len(outs)]
        yuv = out in cc.YUV420
        W, H = int(rng.integers(16, 48)), int(rng.integers(12, 36))
        recolor = yuv and t % 3 == 0
        dst_color = [3, 1, 1] if recolor else None                     # BT709, 0-255, chroma site NONE
        n = int(rng.integers(2, 6))
        pads, spec, keep = (ob.OraclePad * n)(), [], []
        i = 0
        while i < n:
            fmt = "BGRx" if recolor else str(rng.choice(cc.IN_FORMATS + (out,) * 2))
            iw, ih = int(rng.integers(4, 40)), int(rng.integers(4, 32))
            w, h = (iw, ih) if fmt == out and i == 0 else (int(rng.integers(2, 36)), int(rng.integers(2, 28)))
            x, y = int(rng.integers(-w // 2, W)), int(rng.integers(-h // 2, H))
            al, op = float(rng.choice([1.0, 0.5, 0.999, 0.004])), int(rng.integers(0, 3))
            seed = int(rng.integers(0, 1 << 30))
            a = cc.random_frame(lib, fmt, iw, ih, seed)
            if fmt != out or (w, h) != (iw, ih):
                om, orr, osite = dst_color if dst_color else (-1, -1, -1)
                if yuv and not dst_color:
                    ref_info = cc.info(lib, out, W, H)
                    om, orr, osite = ref_info.color_matrix, ref_info.color_range, ref_info.chroma_site
                conv = ob.RefVcs(iw, ih, w, h, -1, in_fmt=cc.FMT[fmt], out_fmt=cc.FMT[out], out_matrix=om, out_rng=orr,
                                 out_site=osite)
                size = o.oracle_compositor_yuv_size(cc.FMT[out], w, h) if yuv else w * h * 4
                ra = conv.convert(a, np.zeros(size, dtype=np.uint8))
                conv.close()
                desc = ob.vcs_desc(iw, ih, w, h, cc.MITCHELL, in_fmt=cc.FMT[fmt], out_fmt=cc.FMT[out])
                if not dst_color and not np.array_equal(ra, ob.oracle_vcs_convert(desc, a)):
                    continue                                            # see the note above: draw this pad again
                a = ra
            keep.append(a)
            pads[i].data, pads[i].width, pads[i].height, pads[i].stride = a.ctypes.data, w, h, 0 if yuv else w * 4
            pads[i].xpos, pads[i].ypos, pads[i].alpha, pads[i].op = x, y, al, op
            spec.append(dict(in_fmt=fmt, iw=iw, ih=ih, pw=w, ph=h, x=x, y=y, alpha=al, op=op, seed=seed, odd=False, kar=False))
            i += 1
        bg = int(rng.integers(0, 4))
        if yuv:
            dst = np.zeros(o.oracle_compositor_yuv_size(cc.FMT[out], W, H), dtype=np.uint8)
            full = dst_color is not None and dst_color[1] == 1
            r.ref_compositor_yuv(cc.FMT[out], dst.ctypes.data, W, H, bg, 0 if full else 1, pads, n)
        else:
            dst = np.zeros(W * H * 4, dtype=np.uint8)
            r.ref_compositor(cc.FMT[out], dst.ctypes.data, W, H, W * 4, bg, pads, n)
        key = f"cc_{t}"
        arrays[key] = cc.unpack(out, dst, cc.info(lib, out, W, H))
        cases.append(dict(key=key, out=out, W=W, H=H, bg=bg, dst_odd=False, dst_color=dst_color, pads=spec))
    np.savez_compressed(os.path.join(HERE, "comp_convert.npz"), **arrays)
    json.dump(cases, open(os.path.join(HERE, "comp_convert_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    assert ob.have_ref(), "needs oracle/_ref/libgstref.so (make -C oracle ref)"
    main()
