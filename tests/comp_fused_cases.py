"""TEST INFRASTRUCTURE: the fused route's plane scalers (b200_comp_blend_convert), form by form.

A 4:2:0 pad whose converter scales planes into the output's format is scaled straight into the compositor's destination
by the CompStore forms of the plane kernels: vcs_planes_comp_kernel (the byte kernel) and the instantiations
vcs_planes_fast[_vfirst]_comp_kernel<H, V, NC, NTW> of plane_fast_kernel_for (vcs_planes_fast.cuh).  H / V: each axis's
pass (1 copy or nearest, 2 two taps, 3 n taps); NC: bytes per pixel (1, or 2 for an interleaved UV plane); NTW: the n-tap
axes' packed tap words (0: run-time loops).

  ROWS         one conversion per reachable form, with the form its convert must launch (read from the emulated launch
               log by tests/test_comp_fused.py)
  UNREACHABLE  every other form the library compiles, with the rule of the plan or of plane_fast_kernel_for that keeps it
               from ever being launched; ROWS and UNREACHABLE together are the library's CompStore kernels
  row_case     four pads of a row's converter sharing one launch, clipping each edge of the destination at odd and negative
               positions, at alphas copy, 254, 128 and 1, their content worst cases of the pad's own taps (worstcase.frame)
  store_case   the full (p, v, a) domain of comp_store through a form whose axes pick source bytes
"""
import re
import subprocess
from collections import namedtuple

import numpy as np

import comp_convert_cases as cc
import comp_domain as cd
import worstcase as wc

Row = namedtuple("Row", "out in_fmt in_size pad_size method odd form")

# (output, pad input, input size, pad size, converter method, input rows at odd strides and offsets, the form it launches)
ROWS = [
    Row("I420", "I420", (100, 9), (200, 18), 0, False, "vcs_planes_comp_kernel"),
    Row("YV12", "YV12", (6, 150), (6, 16), 0, False, "vcs_planes_fast_comp_kernel<1, 1, 1, 0>"),
    Row("NV12", "NV12", (128, 9), (256, 9), 0, False, "vcs_planes_fast_comp_kernel<1, 1, 2, 0>"),
    Row("YV12", "YV12", (150, 9), (150, 24), 1, False, "vcs_planes_fast_comp_kernel<1, 2, 1, 0>"),
    Row("NV12", "NV12", (24, 200), (24, 100), 1, False, "vcs_planes_fast_comp_kernel<1, 2, 2, 0>"),
    Row("YV12", "YV12", (17, 100), (17, 48), 3, False, "vcs_planes_fast_comp_kernel<1, 3, 1, 0>"),
    Row("I420", "I420", (96, 8), (96, 200), 2, False, "vcs_planes_fast_comp_kernel<1, 3, 1, 1>"),
    Row("NV21", "NV21", (300, 128), (300, 8), 3, False, "vcs_planes_fast_comp_kernel<1, 3, 2, 0>"),
    Row("NV12", "NV12", (96, 256), (96, 24), 2, False, "vcs_planes_fast_comp_kernel<1, 3, 2, 1>"),
    Row("YV12", "YV12", (24, 3), (64, 3), 1, False, "vcs_planes_fast_comp_kernel<2, 1, 1, 0>"),
    Row("I420", "I420", (24, 17), (96, 200), 1, False, "vcs_planes_fast_comp_kernel<2, 2, 1, 0>"),
    Row("YV12", "YV12", (24, 17), (200, 8), 3, False, "vcs_planes_fast_comp_kernel<2, 3, 1, 0>"),
    Row("I420", "I420", (16, 8), (32, 4), 2, False, "vcs_planes_fast_comp_kernel<2, 3, 1, 1>"),
    Row("YV12", "YV12", (96, 33), (3, 33), 3, False, "vcs_planes_fast_comp_kernel<3, 1, 1, 0>"),
    Row("I420", "I420", (256, 24), (128, 24), 2, False, "vcs_planes_fast_comp_kernel<3, 1, 1, 1>"),
    Row("NV21", "NV21", (100, 2), (32, 4), 3, False, "vcs_planes_fast_comp_kernel<3, 1, 2, 0>"),
    Row("NV12", "NV12", (100, 32), (256, 32), 1, False, "vcs_planes_fast_comp_kernel<3, 1, 2, 1>"),
    Row("YV12", "YV12", (64, 2), (32, 200), 3, False, "vcs_planes_fast_comp_kernel<3, 2, 1, 0>"),
    Row("I420", "I420", (5, 17), (2, 100), 2, False, "vcs_planes_fast_comp_kernel<3, 2, 1, 1>"),
    Row("NV21", "NV21", (200, 33), (5, 66), 3, False, "vcs_planes_fast_comp_kernel<3, 2, 2, 0>"),
    Row("NV12", "NV12", (8, 9), (17, 200), 1, False, "vcs_planes_fast_comp_kernel<3, 2, 2, 1>"),
    Row("YV12", "YV12", (150, 16), (128, 8), 3, False, "vcs_planes_fast_comp_kernel<3, 3, 1, 0>"),
    Row("I420", "I420", (3, 33), (6, 66), 2, False, "vcs_planes_fast_comp_kernel<3, 3, 1, 1>"),
    Row("NV21", "NV21", (33, 24), (66, 2), 3, False, "vcs_planes_fast_comp_kernel<3, 3, 2, 0>"),
    Row("NV12", "NV12", (520, 12), (33, 8), 2, False, "vcs_planes_fast_comp_kernel<3, 3, 2, 1>"),
    Row("YV12", "YV12", (33, 48), (16, 2), 0, False, "vcs_planes_fast_vfirst_comp_kernel<1, 1, 1, 0>"),
    Row("NV12", "NV12", (300, 300), (150, 17), 0, False, "vcs_planes_fast_vfirst_comp_kernel<1, 1, 2, 0>"),
    Row("YV12", "YV12", (2, 520), (3, 150), 1, False, "vcs_planes_fast_vfirst_comp_kernel<1, 2, 1, 0>"),
    Row("NV12", "NV12", (2, 9), (24, 4), 1, False, "vcs_planes_fast_vfirst_comp_kernel<1, 2, 2, 0>"),
    Row("YV12", "YV12", (2, 150), (4, 16), 3, False, "vcs_planes_fast_vfirst_comp_kernel<1, 3, 1, 0>"),
    Row("I420", "I420", (2, 300), (16, 128), 2, False, "vcs_planes_fast_vfirst_comp_kernel<1, 3, 1, 1>"),
    Row("YV12", "YV12", (2, 33), (4, 16), 3, False, "vcs_planes_fast_vfirst_comp_kernel<1, 3, 1, 2>"),
    Row("NV12", "NV12", (2, 256), (4, 48), 3, False, "vcs_planes_fast_vfirst_comp_kernel<1, 3, 2, 0>"),
    Row("NV21", "NV21", (2, 300), (520, 12), 2, False, "vcs_planes_fast_vfirst_comp_kernel<1, 3, 2, 1>"),
    Row("NV12", "NV12", (2, 24), (4, 9), 4, False, "vcs_planes_fast_vfirst_comp_kernel<1, 3, 2, 2>"),
    Row("YV12", "YV12", (96, 64), (33, 2), 1, False, "vcs_planes_fast_vfirst_comp_kernel<2, 2, 1, 0>"),
    Row("I420", "I420", (4, 96), (24, 12), 3, False, "vcs_planes_fast_vfirst_comp_kernel<2, 3, 1, 0>"),
    Row("YV12", "YV12", (48, 150), (128, 75), 2, False, "vcs_planes_fast_vfirst_comp_kernel<2, 3, 1, 1>"),
    Row("I420", "I420", (6, 300), (12, 96), 3, False, "vcs_planes_fast_vfirst_comp_kernel<2, 3, 1, 2>"),
    Row("NV21", "NV21", (150, 16), (200, 5), 1, False, "vcs_planes_fast_vfirst_comp_kernel<3, 2, 2, 1>"),
    Row("I420", "I420", (6, 300), (12, 96), 3, False, "vcs_planes_fast_vfirst_comp_kernel<3, 3, 1, 0>"),
    Row("YV12", "YV12", (520, 64), (48, 17), 2, False, "vcs_planes_fast_vfirst_comp_kernel<3, 3, 1, 1>"),
    Row("I420", "I420", (48, 300), (33, 150), 3, False, "vcs_planes_fast_vfirst_comp_kernel<3, 3, 1, 2>"),
    Row("NV21", "NV21", (24, 256), (100, 9), 3, False, "vcs_planes_fast_vfirst_comp_kernel<3, 3, 2, 0>"),
    Row("NV12", "NV12", (200, 32), (400, 2), 2, False, "vcs_planes_fast_vfirst_comp_kernel<3, 3, 2, 1>"),
    Row("NV21", "NV21", (64, 33), (16, 16), 3, False, "vcs_planes_fast_vfirst_comp_kernel<3, 3, 2, 2>"),
    Row("I420", "I420", (48, 40), (40, 30), 9, True, "vcs_planes_comp_kernel"),
]


def unreachable_reason(form):
    """why the library never launches `form`, or None when some conversion does"""
    m = re.fullmatch(r"vcs_planes_fast(_vfirst)?_comp_kernel<(\d), (\d), (\d), (\d)>", form)
    if not m:
        return None
    vfirst, (H, V, NC, NTW) = bool(m.group(1)), (int(x) for x in m.groups()[1:])
    if NTW > 0 and 3 not in (H, V):
        return "NTW > 0 needs an n-tap axis (plane_fast_kernel_for picks NTW > 0 only when H or V is 3)"
    if H == 2 and NC == 2:
        return ("H = 2 is the stepping 2-tap scaler of 1-byte planes only (build_planes: two_tap_stepping = ne == 1); a "
                "2-tap interleaved UV axis is an n-tap axis")
    if vfirst and V == 1 and H != 1:
        return ("vertical-first needs both axes scaled and the vertical one shrinking (build_planes: h_first); a 1-tap "
                "vertical axis is either the nearest filter, which makes the horizontal axis 1-tap too, or a 1-line "
                "plane, which cannot shrink")
    if vfirst and H == 3 and V == 2 and (NC, NTW) != (2, 1):
        return ("a shrinking axis has 2 taps only under the 2-tap bilinear method, which makes a 1-byte plane's "
                "horizontal axis the stepping 2-tap scaler (H = 2) and a UV plane's an n-tap axis of one tap word (NTW 1)")
    return None


def library_forms(path):
    """the CompStore kernels in the library's symbol table"""
    out = subprocess.run(["nm", "-C", path], capture_output=True, text=True, check=True).stdout
    return set(re.findall(r"b200::(vcs_planes\w*_comp_kernel(?:<[^>]*>)?)", out))


def content(method, out):
    """per pad: a worst-case frame of its own conversion (the FIR saturates before comp_store blends)"""
    def frame(p):
        return wc.frame(p["in_fmt"], out, (p["iw"], p["ih"], p["pw"], p["ph"]), method, p["seed"])
    return frame


ALPHAS = (1.0, cd.alpha_for(254, 255), cd.alpha_for(128, 255), cd.alpha_for(1, 255))


def row_case(row, seed=0):
    """four pads of the row's converter: each clips one corner of the destination at odd, negative or past-the-edge
    positions, at alphas copy, 254, 128 and 1, all disjoint (one launch); under them the background"""
    (iw, ih), (pw, ph) = row.in_size, row.pad_size
    W, H = 2 * pw + 7, 2 * ph + 7
    cx, cy = min(3, pw - 2) if pw > 2 else -1, min(5, ph - 2) if ph > 2 else -1    # past the edge, some of the pad left
    pos = [(-cx, -cy), (W - pw + cx, -1), (-1, H - ph + cy), (W - pw + 1, H - ph + cy)]
    pads = [cc.pad(row.in_fmt, iw, ih, pw, ph, x, y, alpha=a, op=cd.OVER, seed=seed + k, odd=row.odd)
            for k, ((x, y), a) in enumerate(zip(pos, ALPHAS))]
    return dict(out=row.out, W=W, H=H, bg=cd.CHECKER, dst_odd=False, pads=pads, method=row.method,
                content=content(row.method, row.out))


# forms whose axes pick source bytes, so that each scaled byte v is a chosen byte: the byte kernel (nearest, exactly 2x:
# plane doubling) and vcs_planes_fast_comp_kernel<1, 1, 1, 0> (nearest, 1x vertically)
STORE_FORMS = {"vcs_planes_comp_kernel": ((256, 128), (512, 256)),
               "vcs_planes_fast_comp_kernel<1, 1, 1, 0>": ((256, 250), (512, 252))}


def store_case(form, alphas):
    """the full (p, v, a) domain of comp_store: pad 0 (I420, no converter, copied) lays destination bytes p, then one
    nearest-scaled I420 pad per alpha over its own band; luma source byte (y, x) is x & 255, and the destination's
    bytes are laid so that every p meets every v in each band"""
    (iw, ih), (pw, ph) = STORE_FORMS[form]
    n = len(alphas)
    W, H = pw, ph * n
    pads = [cc.pad("I420", W, H, W, H, 0, 0, alpha=1.0, op=cd.SOURCE, seed=0)]
    pads += [cc.pad("I420", iw, ih, pw, ph, 0, k * ph, alpha=a, op=cd.OVER, seed=1 + k) for k, a in enumerate(alphas)]

    def frame(p):
        y, x = np.mgrid[0:p["ih"], 0:p["iw"]]
        cy, cx = y[::2, ::2], x[::2, ::2]
        if p["seed"] == 0:                                          # the destination's bytes p: every p under every v
            luma = ((x // 2) * 7 + (y % ph) * 2 + (x & 1)) & 255
        else:                                                       # the source: luma byte = its column
            luma = x & 255
        c = (cx * 5 + cy * (3 if p["seed"] else 1)) & 255
        return np.concatenate([luma.ravel(), c.ravel(), (255 - c).ravel()]).astype(np.uint8)
    return dict(out="I420", W=W, H=H, bg=cd.BLACK, dst_odd=False, pads=pads, method=0, content=frame)
