#!/usr/bin/env python
"""bench_extra.py — secondary BASELINE configs on one GPU (kernel-resident numbers):
  C1  cudavideoconvertscale: 1080p NV12 -> 720p BGRA, bilinear (configs[0], the element default)
  C4  cudacompositor: 16 x 1080p RGBA pads -> 3840x2160 RGBA   (configs[3])
  C5  cudaaudioresample: 48k -> 44.1k F32, 256 channels          (configs[4], shortened buffer)
Prints one JSON line per config with achieved GB/s against the measured HBM peak and, for C5,
achieved non-FMA FP32 GFLOP/s (the binding resource, SURVEY §8d)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


QUIET = False      # bench.py imports these benches and embeds their results instead of printing them


def emit(d):
    if not QUIET:
        print(json.dumps(d), flush=True)
    return d


def peak():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 6650.0


def bench_c1(args):
    import numpy as np
    import torch
    import gstreamer_b200 as g
    from oracle import bindings as ob
    IW, IH, OW, OH = 1920, 1080, 1280, 720
    el = g.CudaVideoConvertScale(method=1)
    ii, oi = g.VideoInfo(g.VideoFormat.NV12, IW, IH), g.VideoInfo(g.VideoFormat.BGRA, OW, OH)
    el.set_info(ii, oi)
    if args.variant >= 0:
        el.set_kernel_variant(args.variant)
    ring, per = 128, 64                       # 128 x (3.1 + 3.7) MB = 870 MB >> L2
    base = [torch.from_numpy(ob.nv12_random_frame(IW, IH, s)).cuda() for s in range(4)]
    rin = []
    for k in range(ring):
        t = base[k % 4].clone()
        t[::4099] = (t[::4099].to(torch.int32) + k).to(torch.uint8)
        rin.append(t)
    rout = [torch.empty(oi.size, dtype=torch.uint8, device="cuda") for _ in range(ring)]
    s = torch.cuda.Stream()
    step = lambda i: el.transform_frames(rin[(i % 2) * per:(i % 2 + 1) * per], rout[(i % 2) * per:(i % 2 + 1) * per], s)
    with torch.cuda.stream(s):
        for i in range(4):
            step(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for i in range(args.steps):
            step(i)
        e1.record(s)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    alg = per * (ii.size + oi.size)
    cpu = None
    if ob.have_ref() and not args.no_cpu:
        for threads in (1, os.cpu_count() or 1):
            conv = ob.RefVcs(IW, IH, OW, OH, 1, n_threads=threads)
            f = ob.nv12_smpte_like_frame(IW, IH) if hasattr(ob, "nv12_smpte_like_frame") else ob.nv12_random_frame(IW, IH, 0)
            out = np.zeros(oi.size, dtype=np.uint8)
            conv.convert(f, out)
            n, t0 = 0, time.perf_counter()
            while time.perf_counter() - t0 < 4:
                conv.convert(f, out)
                n += 1
            fps = n / (time.perf_counter() - t0)
            if threads == 1:
                cpu = {"value": fps, "unit": "frames/s", "cores": 1, "kind": "reference",
                       "sample": f"{n} frames, video-converter.c + ORC C backups, n-threads=1 (element default)"}
            else:
                cpu["all_cores"] = {"value": fps, "cores": threads}
    return emit({"config": "C1 cudavideoconvertscale 1920x1080 NV12 -> 1280x720 BGRA bilinear",
                      "kernel_variant": int(el.plan_info().kernel_variant),
                      "frames_per_s": per * 1e3 / ms, "us_per_frame": ms * 1e3 / per,
                      "mpix_per_s_in": per * IW * IH / (ms * 1e-3) / 1e6,
                      "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peak(), "unit": "GB/s",
                                   "frac": alg / (ms * 1e-3) / 1e9 / peak(), "alg_bytes_per_launch": alg},
                      "cpu_baseline": cpu})


def bench_ntap(args):
    """not a BASELINE config: lanczos at ratios the 2:1 kernel does not take (n-tap kernel vs generic)"""
    import torch
    import gstreamer_b200 as g
    from oracle import bindings as ob
    for (IW, IH, OW, OH) in [(1920, 1080, 1280, 720), (3840, 2160, 1280, 720), (1280, 720, 1920, 1080)]:
        el = g.CudaVideoConvertScale(method=3)
        ii, oi = g.VideoInfo(g.VideoFormat.NV12, IW, IH), g.VideoInfo(g.VideoFormat.BGRA, OW, OH)
        el.set_info(ii, oi)
        if args.variant >= 0:
            el.set_kernel_variant(args.variant)
        per = 32
        base = [torch.from_numpy(ob.nv12_random_frame(IW, IH, s)).cuda() for s in range(2)]
        rin = [base[k % 2].clone() for k in range(2 * per)]
        rout = [torch.empty(oi.size, dtype=torch.uint8, device="cuda") for _ in range(2 * per)]
        s = torch.cuda.Stream()
        step = lambda i: el.transform_frames(rin[(i % 2) * per:(i % 2 + 1) * per], rout[(i % 2) * per:(i % 2 + 1) * per], s)
        with torch.cuda.stream(s):
            for i in range(3):
                step(i)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for i in range(args.steps):
                step(i)
            e1.record(s)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        alg = per * (ii.size + oi.size)
        print(json.dumps({"config": f"lanczos {IW}x{IH} NV12 -> {OW}x{OH} BGRA", "kernel_variant": int(el.plan_info().kernel_variant),
                          "us_per_frame": ms * 1e3 / per, "frames_per_s": per * 1e3 / ms,
                          "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peak(), "unit": "GB/s",
                                       "frac": alg / (ms * 1e-3) / 1e9 / peak()}}), flush=True)


def bench_planes(args):
    """not a BASELINE config: YUV -> YUV plane scaling (the transcoding-ladder case)"""
    import torch
    import gstreamer_b200 as g
    from oracle import bindings as ob
    # (input format, output format, ...): 23 NV12, 2 I420; a differing pair is the cross-family chain (two launches)
    results = []
    for (fmt, fmt_o, IW, IH, OW, OH, m) in [(23, 23, 3840, 2160, 1920, 1080, 1), (23, 23, 3840, 2160, 1920, 1080, 3),
                                            (2, 2, 1920, 1080, 1280, 720, 3), (23, 23, 1920, 1080, 1280, 720, 1),
                                            (23, 2, 3840, 2160, 1920, 1080, 3), (23, 2, 1920, 1080, 1280, 720, 1),
                                            (12, 12, 3840, 2160, 1920, 1080, 1), (12, 11, 3840, 2160, 1920, 1080, 3),
                                            (12, 12, 1920, 1080, 1280, 720, 3),       # 12 BGRA, 11 RGBA: 4-byte pixels
                                            (12, 23, 1920, 1080, 1920, 1080, 1), (12, 23, 3840, 2160, 3840, 2160, 1),
                                            (12, 23, 3840, 2160, 1920, 1080, 1), (12, 23, 3840, 2160, 1920, 1080, 3),
                                            (11, 2, 1920, 1080, 1280, 720, 3), (12, 23, 1280, 720, 1920, 1080, 1),      # compositor output -> encoder input
                                            (4, 2, 1920, 1080, 1920, 1080, 1), (4, 23, 1920, 1080, 1920, 1080, 1)]:   # capture (YUY2) -> encoder input
        el = g.CudaVideoConvertScale(method=m)
        ii, oi = g.VideoInfo(fmt, IW, IH), g.VideoInfo(fmt_o, OW, OH)
        if fmt != fmt_o:                              # what the element's caps fixation does for YUV -> YUV
            from gstreamer_b200.video import transfer_colorimetry_from_input
            transfer_colorimetry_from_input(ii, oi)
        el.set_info(ii, oi)
        per = 32
        if fmt in (11, 12, 4, 5):
            import numpy as np
            gen = lambda w, h, seed, nbytes=ii.size: np.random.default_rng(seed).integers(0, 256, nbytes, dtype=np.uint8)
        else:
            gen = ob.i420_random_frame if fmt in (2, 3) else ob.nv12_random_frame
        base = [torch.from_numpy(gen(IW, IH, s)).cuda() for s in range(2)]
        rin = [base[k % 2].clone() for k in range(2 * per)]
        rout = [torch.empty(oi.size, dtype=torch.uint8, device="cuda") for _ in range(2 * per)]
        s = torch.cuda.Stream()
        step = lambda i: el.transform_frames(rin[(i % 2) * per:(i % 2 + 1) * per], rout[(i % 2) * per:(i % 2 + 1) * per], s)
        with torch.cuda.stream(s):
            for i in range(3):
                step(i)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for i in range(args.steps):
                step(i)
            e1.record(s)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        alg = per * (ii.size + oi.size)
        results.append(emit({"config": f"{g.VideoFormat(fmt).name} {IW}x{IH} -> {g.VideoFormat(fmt_o).name} {OW}x{OH} method {m}",
                             "kernel_variant": int(el.plan_info().kernel_variant), "us_per_frame": ms * 1e3 / per,
                             "frames_per_s": per * 1e3 / ms,
                             "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peak(), "unit": "GB/s",
                                          "frac": alg / (ms * 1e-3) / 1e9 / peak(), "alg_bytes_per_launch": alg}}))
        del rin, rout, base
    return results


def bench_audio_formats(args):
    """C5 shape (48k -> 44.1k, 256 channels, 20 s buffer) in the other sample formats (correctness-first kernels)"""
    import torch
    from gstreamer_b200.audio import CudaAudioResample, AudioFormat
    ch, in_rate, out_rate, seconds = 256, 48000, 44100, 5
    frames = in_rate * seconds
    for name, fmt, tdt in [("S16", AudioFormat.S16LE, torch.int16), ("S32", AudioFormat.S32LE, torch.int32),
                           ("F64", AudioFormat.F64LE, torch.float64)]:
        rs = CudaAudioResample(quality=4, format=fmt)
        rs.set_caps(in_rate, out_rate, ch)
        if tdt.is_floating_point:
            x = torch.randn(frames * ch, dtype=tdt, device="cuda") * 0.25
        else:
            x = torch.randint(-20000, 20000, (frames * ch,), dtype=tdt, device="cuda")
        cap = int(frames * out_rate / in_rate) + 64
        out = torch.empty(cap * ch, dtype=tdt, device="cuda")
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            rs.transform(x, frames, out, cap, stream=s)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for _ in range(3):
                rs.reset()
                rs.transform(x, frames, out, cap, stream=s)
            e1.record(s)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 3
        print(json.dumps({"config": f"cudaaudioresample 48k->44.1k {name} 256ch, {seconds} s buffer", "ms_per_buffer": ms,
                          "realtime_factor": seconds / (ms * 1e-3)}), flush=True)


def bench_c4(args):
    import numpy as np
    import torch
    from gstreamer_b200.compositor import CudaCompositor
    from oracle import bindings as ob
    W, H = 3840, 2160
    rng = np.random.default_rng(0)
    out_ring = [torch.empty(W * H * 4, dtype=torch.uint8, device="cuda") for _ in range(6)]
    rings = []
    for ring in range(3):            # 3 sets of 16 pads = 398 MB of sources, > L2
        comp = CudaCompositor(11, W, H, args.background)
        for k in range(16):
            src = torch.randint(0, 256, (1080 * 1920 * 4,), dtype=torch.uint8, device="cuda")
            comp.request_pad(1920, 1080, xpos=(k % 4) * 640, ypos=(k // 4) * 360,
                             alpha=0.5 if k % 2 else 1.0).set_frame(src)
        rings.append(comp)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for i in range(5):
            rings[i % 3].aggregate_frames(out_ring[i % 6], stream=s)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for i in range(args.steps):
            rings[i % 3].aggregate_frames(out_ring[i % 6], stream=s)
        e1.record(s)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    alg = 16 * 1920 * 1080 * 4 + W * H * 4
    # CPU baseline: the reference's blend.c on one frame
    cpu = None
    if ob.have_ref() and not args.no_cpu:
        r = ob.ref()
        pads = (ob.OraclePad * 16)()
        keep = []
        for k in range(16):
            a = rng.integers(0, 256, (1080, 1920, 4), dtype=np.uint8)
            keep.append(a)
            pads[k].data, pads[k].width, pads[k].height, pads[k].stride = a.ctypes.data, 1920, 1080, 7680
            pads[k].xpos, pads[k].ypos, pads[k].alpha, pads[k].op = (k % 4) * 640, (k // 4) * 360, 0.5 if k % 2 else 1.0, 1
        dst = np.zeros((H, W, 4), dtype=np.uint8)
        r.ref_compositor(11, dst.ctypes.data, W, H, W * 4, args.background, pads, 16)
        t0 = time.perf_counter()
        n = 0
        while time.perf_counter() - t0 < 5:
            r.ref_compositor(11, dst.ctypes.data, W, H, W * 4, args.background, pads, 16)
            n += 1
        cpu = {"value": n / (time.perf_counter() - t0), "unit": "frames/s", "cores": 1, "kind": "reference",
               "sample": f"{n} frames, blend.c + ORC C backups, single thread"}
    return emit({"config": "C4 cudacompositor 16x1080p RGBA -> 4K RGBA", "background": args.background,
                      "frames_per_s": 1e3 / ms, "us_per_frame": ms * 1e3,
                      "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peak(), "unit": "GB/s",
                                   "frac": alg / (ms * 1e-3) / 1e9 / peak(), "alg_bytes_per_launch": alg},
                      "cpu_baseline": cpu})


def bench_c5(args):
    import numpy as np
    import torch
    from gstreamer_b200.audio import CudaAudioResample
    from oracle import bindings as ob
    ch, in_rate, out_rate = 256, 48000, 44100
    frames = in_rate * args.seconds
    rs = CudaAudioResample(quality=4)
    rs.set_caps(in_rate, out_rate, ch)
    x = torch.randn(frames * ch, dtype=torch.float32, device="cuda") * 0.25
    cap = int(frames * out_rate / in_rate) + 64
    out = torch.empty(cap * ch, dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(2):
            rs.reset()
            rs.transform(x, frames, out, cap, stream=s)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n_out = 0
        e0.record(s)
        for _ in range(args.steps):
            n_out = rs.transform(x, frames, out, cap, stream=s)
        e1.record(s)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    taps = rs.plan_info().n_taps
    alg = (frames + n_out) * ch * 4
    flops = 2.0 * taps * n_out * ch
    cpu = None
    if ob.have_ref() and not args.no_cpu:
        r = ob.ref()
        h = r.ref_ars_new(in_rate, out_rate, ch, 4)
        n = in_rate // 2
        xi = (np.random.default_rng(0).standard_normal((n, ch)) * 0.25).astype(np.float32)
        o = np.zeros((n, ch), dtype=np.float32)
        r.ref_ars_process(h, xi.ctypes.data, n, o.ctypes.data, n)
        t0 = time.perf_counter()
        k = 0
        while time.perf_counter() - t0 < 5:
            r.ref_ars_process(h, xi.ctypes.data, n, o.ctypes.data, n)
            k += 1
        dt = time.perf_counter() - t0
        cpu = {"value": k * n * ch / dt / 1e6, "unit": "Msamples/s (input)", "cores": 1, "kind": "reference",
               "sample": f"{k} x 0.5 s buffers, audio-resampler.c SSE inner product, single thread"}
        r.ref_ars_free(h)
    return emit({"config": f"C5 cudaaudioresample 48k->44.1k F32 256ch, {args.seconds} s buffer",
                      "msamples_per_s_in": frames * ch / (ms * 1e-3) / 1e6, "ms_per_buffer": ms,
                      "realtime_factor": args.seconds / (ms * 1e-3),
                      "roofline": {"bound": "fp32-issue (no FMA allowed for bit-exactness), then hbm",
                                   "achieved": alg / (ms * 1e-3) / 1e9, "peak": peak(), "unit": "GB/s",
                                   "frac": alg / (ms * 1e-3) / 1e9 / peak(),
                                   "achieved_gflops": flops / (ms * 1e-3) / 1e9, "alg_bytes_per_launch": alg},
                      "cpu_baseline": cpu})


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--seconds", type=int, default=20)
    ap.add_argument("--background", type=int, default=0)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--only", default="")
    ap.add_argument("--variant", type=int, default=-1, help="C1: force a convert+scale kernel variant")
    a = ap.parse_args()
    if a.only in ("", "c1"):
        bench_c1(a)
    if a.only == "audiofmt":
        bench_audio_formats(a)
    if a.only == "planes":
        bench_planes(a)
    if a.only == "ntap":
        bench_ntap(a)
    if a.only in ("", "c4"):
        bench_c4(a)
    if a.only in ("", "c5"):
        bench_c5(a)
