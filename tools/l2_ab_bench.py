#!/usr/bin/env python
"""tools/l2_ab_bench.py — two (or more) builds of libb200dsp.so against each other on the 2:1 Lanczos shapes, alternated.

    python tools/l2_ab_bench.py --lib base=build/baseline/libb200dsp.so --lib new=gstreamer_b200/libb200dsp.so

Every build is loaded by path with its own ctypes binding (gstreamer_b200/_lib.py binds one fixed path), gets its own
converter handle, and runs the workload of bench.py: a ring of 64 distinct frames resident in HBM, 32 frames per launch,
CUDA events around a round of launches.  Rounds alternate between the builds (A B A B ...), so clock drift and other
tenants of the host hit every build alike.  Printed per shape: us/frame of every round, each build's median and spread
(max - min over its rounds), the SM clock median NVML reported during each build's rounds, and whether the builds' outputs
are byte-identical.  The card's name and power limit are read (never set) and printed with the numbers.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from gstreamer_b200._lib import VideoInfoC, VcsConfigC  # noqa: E402  (struct layouts only)
from oracle import bindings as ob  # noqa: E402  (input generator only)

NV12, I420, BGRA, LANCZOS = 23, 2, 12, 3
SHAPES = {
    "bench": ("3840x2160 NV12 -> 1920x1080 BGRA", NV12, 3840, 2160, 1920, 1080),
    "i420": ("3840x2160 I420 -> 1920x1080 BGRA", I420, 3840, 2160, 1920, 1080),
    "1080p": ("1920x1080 NV12 -> 960x540 BGRA", NV12, 1920, 1080, 960, 540),
}
RING, PER = 64, 32
_P = C.c_void_p


class Build:
    """the C-ABI calls this script needs, bound on one build of the library"""

    def __init__(self, name, path):
        self.name, self.lib = name, C.CDLL(os.path.abspath(path))
        L = self.lib
        L.b200_video_info_set_format.restype, L.b200_video_info_set_format.argtypes = C.c_int, [C.POINTER(VideoInfoC), C.c_int, C.c_int, C.c_int]
        L.b200_video_info_size.restype, L.b200_video_info_size.argtypes = C.c_size_t, [C.POINTER(VideoInfoC)]
        L.b200_vcs_config_init.restype, L.b200_vcs_config_init.argtypes = None, [C.POINTER(VcsConfigC)]
        L.b200_vcs_create.restype = C.c_int
        L.b200_vcs_create.argtypes = [C.POINTER(VideoInfoC), C.POINTER(VideoInfoC), C.POINTER(VcsConfigC), C.c_int, C.POINTER(_P)]
        L.b200_vcs_convert_batch.restype, L.b200_vcs_convert_batch.argtypes = C.c_int, [_P, C.c_int, C.POINTER(_P), C.POINTER(_P), _P]
        L.b200_vcs_kernel_name.restype, L.b200_vcs_kernel_name.argtypes = C.c_char_p, [_P]
        L.b200_vcs_destroy.restype, L.b200_vcs_destroy.argtypes = None, [_P]
        self.h = None

    def ok(self, st, what):
        if st < 0:
            raise RuntimeError(f"{self.name}: {what} returned {st}")

    def create(self, fmt, iw, ih, ow, oh):
        ii, oi, cfg, h = VideoInfoC(), VideoInfoC(), VcsConfigC(), _P()
        self.ok(self.lib.b200_video_info_set_format(C.byref(ii), fmt, iw, ih), "b200_video_info_set_format")
        self.ok(self.lib.b200_video_info_set_format(C.byref(oi), BGRA, ow, oh), "b200_video_info_set_format")
        self.lib.b200_vcs_config_init(C.byref(cfg))
        cfg.method = LANCZOS
        self.ok(self.lib.b200_vcs_create(C.byref(ii), C.byref(oi), C.byref(cfg), 0, C.byref(h)), "b200_vcs_create")
        self.h = h
        return self.lib.b200_video_info_size(C.byref(ii)), self.lib.b200_video_info_size(C.byref(oi))

    def kernel(self):
        return self.lib.b200_vcs_kernel_name(self.h).decode()

    def convert(self, ins, outs, stream):
        self.ok(self.lib.b200_vcs_convert_batch(self.h, len(ins), ins, outs, stream), "b200_vcs_convert_batch")

    def destroy(self):
        self.lib.b200_vcs_destroy(self.h)
        self.h = None


class ClockSampler:
    """SM clock during a round: NVML every millisecond, or nvidia-smi queries where pynvml is not installed"""

    def __init__(self):
        self.mhz, self._stop, self._t = [], threading.Event(), None

    def _run(self):
        try:
            import pynvml as nv
            nv.nvmlInit()
            h = nv.nvmlDeviceGetHandleByIndex(int((os.environ.get("CUDA_VISIBLE_DEVICES") or "0").split(",")[0]))
            while not self._stop.is_set():
                self.mhz.append(float(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)))
                self._stop.wait(0.001)
        except Exception:
            while not self._stop.is_set():
                self.mhz.extend(float(v) for v in smi("clocks.sm") if v.replace(".", "").isdigit())
                self._stop.wait(0.02)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join(timeout=6)


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=5).stdout.strip().splitlines()
        return [f.strip() for f in out[0].split(",")] if out else []
    except Exception:
        return []


def run_shape(key, builds, rounds, launches, warmup):
    what, fmt, iw, ih, ow, oh = SHAPES[key]
    gen = ob.i420_random_frame if fmt == I420 else ob.nv12_random_frame
    base = [torch.from_numpy(gen(iw, ih, s)).cuda() for s in range(4)]
    ring_in = []
    for k in range(RING):
        t = base[k % 4].clone()
        t[::4099] = (t[::4099].to(torch.int32) + k).to(torch.uint8)      # every frame distinct, as in bench.py
        ring_in.append(t)
    stream = torch.cuda.Stream()
    state = {}
    for b in builds:
        isz, osz = b.create(fmt, iw, ih, ow, oh)
        assert isz == ring_in[0].numel(), (isz, ring_in[0].numel())
        outs = [torch.zeros(osz, dtype=torch.uint8, device="cuda") for _ in range(RING)]
        args = []
        for o in range(0, RING, PER):
            args.append(((_P * PER)(*[t.data_ptr() for t in ring_in[o:o + PER]]), (_P * PER)(*[t.data_ptr() for t in outs[o:o + PER]])))
        state[b.name] = (outs, args)
        for i in range(warmup):
            b.convert(*args[i % len(args)], stream.cuda_stream)
    torch.cuda.synchronize()
    ref = state[builds[0].name][0]
    same = {b.name: all(torch.equal(x, y) for x, y in zip(ref, state[b.name][0])) for b in builds[1:]}

    us = {b.name: [] for b in builds}
    mhz = {b.name: [] for b in builds}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for b in builds:
            args = state[b.name][1]
            with ClockSampler() as cs:
                e0.record(stream)
                for i in range(launches):
                    b.convert(*args[i % len(args)], stream.cuda_stream)
                e1.record(stream)
                torch.cuda.synchronize()
            us[b.name].append(e0.elapsed_time(e1) * 1e3 / (launches * PER))
            mhz[b.name].extend(cs.mhz)
    res = {"shape": what, "frames_per_launch": PER, "launches_per_round": launches, "rounds": rounds, "builds": {}}
    for b in builds:
        v = us[b.name]
        res["builds"][b.name] = {"kernel": b.kernel(), "us_per_frame_rounds": [round(x, 3) for x in v],
                                 "median_us": round(statistics.median(v), 3), "spread_us": round(max(v) - min(v), 3),
                                 "sm_mhz_median": statistics.median(mhz[b.name]) if mhz[b.name] else None}
        b.destroy()
    m0 = res["builds"][builds[0].name]["median_us"]
    for b in builds[1:]:
        r = res["builds"][b.name]
        r["vs_" + builds[0].name] = f"{(m0 - r['median_us']) / m0 * 100:+.2f}% time saved"
        r["output_identical_to_" + builds[0].name] = same[b.name]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", metavar="NAME=PATH", help="a build of libb200dsp.so; give at least two, the first is the baseline")
    ap.add_argument("--shapes", default="bench,i420,1080p")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    libs = a.lib or ["base=build/baseline/libb200dsp.so", "new=gstreamer_b200/libb200dsp.so"]
    if len(libs) < 2 or a.rounds < 1 or a.launches < 1:
        ap.error("need at least two --lib NAME=PATH and positive --rounds / --launches")
    builds = [Build(*s.split("=", 1)) for s in libs]
    card = smi("name,power.limit,clocks.max.sm")
    print(json.dumps({"card": card[0] if card else torch.cuda.get_device_name(0), "power_limit_w": card[1] if len(card) > 1 else None,
                      "sm_max_mhz": card[2] if len(card) > 2 else None}), flush=True)
    for key in a.shapes.split(","):
        print(json.dumps(run_shape(key, builds, a.rounds, a.launches, max(a.warmup, 5))), flush=True)


if __name__ == "__main__":
    main()
