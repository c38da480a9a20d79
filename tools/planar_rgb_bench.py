#!/usr/bin/env python
"""Planar RGB output (RGBP) against packed BGRx, and against BGRx followed by torch's de-interleave (what users of a
network's (3, H, W) input do without RGBP).  Prints one JSON line.

    python tools/planar_rgb_bench.py [--rounds 7] [--batches 4] [--warmup 2]

Shapes: C2 (3840x2160 NV12 -> 1920x1080, lanczos), C1 (1920x1080 NV12 -> 1280x720, bilinear) and 1920x1080 NV12 -> 640x640
lanczos (an n-tap shape).  Each launch converts 32 frames (b200_vcs_convert_batch); inputs and outputs walk rings of at least
1.3 GB so frames come from HBM, not L2.  The three forms are timed alternately in the same process with CUDA events; the
reported time is the median over rounds (min and max beside it).  Bytes are algorithmic (what each form must read and
write per frame), and the HBM fraction is relative to the H100 SXM data-sheet 3.35 TB/s.  GPU name, power limit and max
SM clock come from read-only NVML queries.  Writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
BATCH = 32
RING_BYTES = 1.3e9
SHAPES = [("C2", 3840, 2160, 1920, 1080, 3), ("C1", 1920, 1080, 1280, 720, 1), ("ntap", 1920, 1080, 640, 640, 3)]


def gpu_facts():
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(int((os.environ.get("CUDA_VISIBLE_DEVICES") or "0").split(",")[0] or 0))
        name = nv.nvmlDeviceGetName(h)
        return {"gpu": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
                "max_sm_clock_mhz": nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM), "source": "nvml"}
    except Exception:
        pass
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1]), "max_sm_clock_mhz": int(out[2]), "source": "nvidia-smi"}
    except Exception:
        return {"gpu": "unknown", "power_limit_w": None, "max_sm_clock_mhz": None, "source": "none"}


def bench_shape(tag, iw, ih, ow, oh, method, rounds, batches, warmup):
    import numpy as np
    import torch
    import gstreamer_b200 as g
    from oracle import bindings as ob

    ii = g.VideoInfo(g.VideoFormat.NV12, iw, ih)
    els = {}
    for fmt in ("RGBP", "BGRx"):
        el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=0)
        oi = g.VideoInfo(g.VideoFormat[fmt], ow, oh)
        el.set_info(ii, oi)
        els[fmt] = (el, oi)
    in_bytes = ii.size
    n_sets = max(2, int(-(-RING_BYTES // (BATCH * in_bytes))))        # ring of input batches >= 1.3 GB
    base = torch.from_numpy(ob.nv12_random_frame(iw, ih, 5)).cuda()
    ins = [[base.clone() for _ in range(BATCH)] for _ in range(n_sets)]
    out_sets = max(2, int(-(-RING_BYTES // (BATCH * els["BGRx"][1].size))))
    outs = {f: [[torch.empty(els[f][1].size, dtype=torch.uint8, device="cuda") for _ in range(BATCH)] for _ in range(out_sets)]
            for f in ("RGBP", "BGRx")}
    chw = [torch.empty((3, oh, ow), dtype=torch.uint8, device="cuda") for _ in range(BATCH)]

    def run(form, k):
        src = ins[k % n_sets]
        if form == "RGBP":
            els["RGBP"][0].transform_frames(src, outs["RGBP"][k % out_sets])
        else:
            dst = outs["BGRx"][k % out_sets]
            els["BGRx"][0].transform_frames(src, dst)
            if form == "BGRx+permute":
                for i in range(BATCH):
                    chw[i].copy_(dst[i].view(oh, ow, 4)[:, :, :3].permute(2, 0, 1))    # = .permute(2, 0, 1).contiguous()

    # correctness of the timed form: RGBP planes are BGRx's R, G, B bytes
    run("RGBP", 0)
    run("BGRx", 0)
    torch.cuda.synchronize()
    a = outs["RGBP"][0][0].view(3, oh, ow).cpu().numpy()
    b = outs["BGRx"][0][0].view(oh, ow, 4).cpu().numpy()
    assert np.array_equal(a, b[:, :, [2, 1, 0]].transpose(2, 0, 1)), f"{tag}: RGBP planes differ from BGRx"

    forms = ("RGBP", "BGRx", "BGRx+permute")
    times = {f: [] for f in forms}
    k = 0
    for f in forms:                                            # warm-up of every form
        for _ in range(warmup * batches):
            run(f, k)
            k += 1
    torch.cuda.synchronize()
    for r in range(rounds):
        order = forms if r % 2 == 0 else forms[::-1]           # alternate, and alternate who goes first
        for f in order:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(batches):
                run(f, k)
                k += 1
            e1.record()
            e1.synchronize()
            times[f].append(e0.elapsed_time(e1) * 1e3 / (batches * BATCH))     # us per frame
    px_in, px_out = iw * ih, ow * oh
    nv12 = in_bytes
    bytes_per_frame = {"RGBP": nv12 + 3 * px_out, "BGRx": nv12 + 4 * px_out, "BGRx+permute": nv12 + 4 * px_out + 4 * px_out + 3 * px_out}
    res = {"shape": tag, "in": [iw, ih], "out": [ow, oh], "method": method, "kernel_rgbp": els["RGBP"][0].kernel_name(),
           "kernel_bgrx": els["BGRx"][0].kernel_name(), "frames_per_launch": BATCH, "input_ring_frames": n_sets * BATCH,
           "forms": {}}
    for f in forms:
        med = statistics.median(times[f])
        res["forms"][f] = {"us_per_frame": round(med, 2), "min": round(min(times[f]), 2), "max": round(max(times[f]), 2),
                           "bytes_per_frame": bytes_per_frame[f],
                           "hbm_fraction": round(bytes_per_frame[f] / (med * 1e-6) / HBM_PEAK, 3)}
    res["rgbp_vs_bgrx"] = round(res["forms"]["RGBP"]["us_per_frame"] / res["forms"]["BGRx"]["us_per_frame"], 3)
    del ins, outs, chw
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--batches", type=int, default=4, help="launches of 32 frames per timed block")
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("planar_rgb_bench: needs a CUDA device")
    facts = gpu_facts()
    shapes = [bench_shape(*s, a.rounds, a.batches, a.warmup) for s in SHAPES]
    print(json.dumps({"bench": "planar_rgb", **facts, "hbm_peak_tbs": HBM_PEAK / 1e12,
                      "hbm_peak_note": "H100 SXM data sheet, not measured", "shapes": shapes}))


if __name__ == "__main__":
    main()
