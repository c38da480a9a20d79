#!/usr/bin/env python
"""tools/comp_mosaic_bench.py [rounds] — the compositor's mosaic workloads on the device, two ways alternated in one process:

  fused     b200_comp_blend_convert (4:2:0 output: the plane scalers store straight into the output frame)
  two-pass  public calls only: b200_vcs_convert_batch into frames, then b200_comp_blend_yuv / b200_comp_blend

  M1  16 x 1920x1080 NV12 pads at 960x540 in a 4 x 4 grid -> 3840x2160 NV12, alpha 1.0, black background
  M2  9 x 1920x1080 NV12 pads at 640x360 in a 3 x 3 grid -> 1920x1080 NV12, plus one more at 640x360, alpha 0.5, on top
      overlapping four tiles
  M3  4 x 1920x1080 NV12 pads at 960x540 -> 1920x1080 BGRA (both ways are two passes; reported, not compared)

CUDA events around 20 calls per timing; the median of the rounds (default 9); inputs in a ring of frame sets larger than
the L2.  Algorithmic bytes: every input frame read once, the output written once.  Prints one JSON line per workload with
the card's name, power limit and max SM clock read in the same run."""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gstreamer_b200 import _lib  # noqa: E402
from gstreamer_b200._lib import lib, check  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
CALLS = 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
        name, power, clock = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:       # the numbers stay; the card is then unknown
        return {"gpu": torch.cuda.get_device_name(0), "card_query_error": str(e)}


def vinfo(fmt, w, h):
    i = _lib.VideoInfoC()
    check(lib.b200_video_info_set_format(C.byref(i), fmt, w, h), "b200_video_info_set_format")
    return i


def workload(name):
    NV12, BGRA = 23, 12
    if name == "M1":
        out, W, H, tiles = NV12, 3840, 2160, [(c * 960, r * 540, 960, 540, 1.0) for r in range(4) for c in range(4)]
    elif name == "M2":
        out, W, H = NV12, 1920, 1080
        tiles = [(c * 640, r * 360, 640, 360, 1.0) for r in range(3) for c in range(3)] + [(320, 180, 640, 360, 0.5)]
    else:
        out, W, H, tiles = BGRA, 1920, 1080, [(c * 960, r * 540, 960, 540, 1.0) for r in range(2) for c in range(2)]
    return out, W, H, tiles


def run(name, rounds):
    out, W, H, tiles = workload(name)
    yuv = out != 12
    n = len(tiles)
    ii = vinfo(23, 1920, 1080)
    fsz = lib.b200_video_info_size(C.byref(ii))
    ring = max(2, int(np.ceil(3 * 50e6 / (n * fsz))))                # frame sets larger than the L2, several times over
    frames = [[torch.randint(0, 256, (fsz,), dtype=torch.uint8, device="cuda") for _ in range(n)] for _ in range(ring)]
    di = vinfo(out, W, H)
    dst = torch.zeros(lib.b200_video_info_size(C.byref(di)), dtype=torch.uint8, device="cuda")
    dst2 = torch.zeros_like(dst)
    comp = C.c_void_p()
    check(lib.b200_comp_create(out, W, H, 0, C.byref(comp)), "b200_comp_create")
    cfg = _lib.VcsConfigC()
    lib.b200_vcs_config_init(C.byref(cfg))
    cfg.method = 9
    convs = {}
    for (_, _, w, h, _) in tiles:                                  # one converter per output size: tiles of a size batch
        if (w, h) not in convs:
            ci = vinfo(out, w, h)
            ci.color_matrix, ci.color_range, ci.chroma_site = di.color_matrix, di.color_range, di.chroma_site
            hv = C.c_void_p()
            check(lib.b200_vcs_create(C.byref(ii), C.byref(ci), C.byref(cfg), 0, C.byref(hv)), "b200_vcs_create")
            convs[(w, h)] = (hv, ci)
    # fused: the pad descriptors of each frame set
    fused_pads = []
    for s in range(ring):
        arr = (_lib.CompPadConvertC * n)()
        for k, (x, y, w, h, a) in enumerate(tiles):
            arr[k].data, arr[k].info, arr[k].conv = frames[s][k].data_ptr(), ii, convs[(w, h)][0]
            arr[k].xpos, arr[k].ypos, arr[k].alpha, arr[k].op = x, y, a, 1
        fused_pads.append(arr)
    # two-pass: converted frames, then the blend of the output's family
    scratch = {k: [torch.empty(lib.b200_video_info_size(C.byref(ci)), dtype=torch.uint8, device="cuda")
                   for (_, _, w, h, _) in tiles if (w, h) == k] for k, (_, ci) in convs.items()}
    blend_pads = (_lib.CompPadYuvC * n)() if yuv else (_lib.CompPadC * n)()
    used = {k: 0 for k in convs}
    for k, (x, y, w, h, a) in enumerate(tiles):
        buf = scratch[(w, h)][used[(w, h)]]
        used[(w, h)] += 1
        blend_pads[k].data = buf.data_ptr()
        if yuv:
            blend_pads[k].info = convs[(w, h)][1]
        else:
            blend_pads[k].width, blend_pads[k].height, blend_pads[k].stride = w, h, convs[(w, h)][1].stride[0]
        blend_pads[k].xpos, blend_pads[k].ypos, blend_pads[k].alpha, blend_pads[k].op = x, y, a, 1
    batches = []
    for s in range(ring):
        per = []
        for key, (hv, _) in convs.items():
            idx = [k for k, t in enumerate(tiles) if (t[2], t[3]) == key]
            ins = (C.c_void_p * len(idx))(*[frames[s][k].data_ptr() for k in idx])
            outs = (C.c_void_p * len(idx))(*[b.data_ptr() for b in scratch[key]])
            per.append((hv, len(idx), ins, outs))
        batches.append(per)

    def fused(s, d):
        check(lib.b200_comp_blend_convert(comp, d.data_ptr(), C.byref(di), 1, fused_pads[s], n, None), "blend_convert")

    def two_pass(s, d):
        for hv, m, ins, outs in batches[s]:
            check(lib.b200_vcs_convert_batch(hv, m, ins, outs, None), "convert_batch")
        if yuv:
            check(lib.b200_comp_blend_yuv(comp, d.data_ptr(), C.byref(di), 1, blend_pads, n, None), "blend_yuv")
        else:
            check(lib.b200_comp_blend(comp, d.data_ptr(), di.stride[0], 1, blend_pads, n, None), "blend")

    fused(0, dst)
    two_pass(0, dst2)
    torch.cuda.synchronize()
    same = bool(torch.equal(dst, dst2))
    times = {"fused": [], "two_pass": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for fn in (fused, two_pass):                                   # warm-up
        for i in range(CALLS):
            fn(i % ring, dst)
    torch.cuda.synchronize()
    for r in range(rounds):
        for key, fn in (("fused", fused), ("two_pass", two_pass)) if r % 2 == 0 else (("two_pass", two_pass), ("fused", fused)):
            ev0.record()
            for i in range(CALLS):
                fn(i % ring, dst)
            ev1.record()
            ev1.synchronize()
            times[key].append(ev0.elapsed_time(ev1) * 1e3 / CALLS)
    in_bytes = n * sum(rb * rows for rb, rows in ((1920, 1080), (1920, 540)))
    out_bytes = W * H * 4 if not yuv else W * H + W * (H // 2)
    alg = in_bytes + out_bytes
    res = {"workload": name, "pads": n, "output": f"{W}x{H} {'NV12' if yuv else 'BGRA'}", "algorithmic_bytes": alg,
           "bytes_identical": same, "rounds": rounds}
    for key, v in times.items():
        us = float(np.median(v))
        res[f"{key}_us"] = round(us, 1)
        res[f"{key}_fraction_of_3.35TBps"] = round(alg / (us * 1e-6) / HBM_BYTES_PER_S, 3)
    for hv, _ in convs.values():
        lib.b200_vcs_destroy(hv)
    lib.b200_comp_destroy(comp)
    return res


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    torch.cuda.init()
    c = card()
    for name in ("M1", "M2", "M3"):
        r = run(name, max(rounds, 7))
        r.update(c)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
