#!/usr/bin/env python
"""cudaaudioresample on packed sample formats: the C5 rate pair (48 kHz -> 44.1 kHz, 256 channels) on a 10 s buffer for
S24LE and S24_32LE (unpacked to S32 inside ars_direct_kernel_packed), S32LE (the same S32 arithmetic in
ars_direct_kernel, no unpack) and F32LE (the tuned persistent pipeline), for context.  The forms alternate in one
process, each call timed with CUDA events, median of 7; the card's name and power limit are read in the same run.
Prints one JSON line per form: us per buffer, x realtime, and the algorithmic bytes (input read once, output written
once) over the time.

    python tools/audio_formats_bench.py [--seconds 10] [--reps 7]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from gstreamer_b200 import _lib  # noqa: E402
from gstreamer_b200._lib import lib, check  # noqa: E402
from gstreamer_b200.audio import AudioFormat  # noqa: E402

FORMS = ["S24LE", "S24_32LE", "S32LE", "F32LE"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
        name, power, clock = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"gpu": torch.cuda.get_device_name(0), "card_query_error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    a, b, ch = 48000, 44100, 256
    n = int(a * args.seconds)
    dev = card()
    handles = {}
    for name in FORMS:
        fmt = getattr(AudioFormat, name)
        cfg = _lib.ArsConfigC()
        cfg.in_rate, cfg.out_rate, cfg.channels, cfg.quality, cfg.format = a, b, ch, 4, fmt
        h = C.c_void_p()
        check(lib.b200_ars_create(C.byref(cfg), 0, C.byref(h)), "b200_ars_create")
        w = AudioFormat.WIDTH[fmt]
        cap = int(lib.b200_ars_get_out_frames(h, n)) + 64
        x = torch.randint(0, 256, (n * ch * w,), dtype=torch.uint8, device="cuda")
        if name == "F32LE":
            x = (torch.randn(n * ch, device="cuda") * 0.3).view(torch.uint8)
        y = torch.empty(cap * ch * w, dtype=torch.uint8, device="cuda")
        handles[name] = (h, x, y, cap, w)
    times = {k: [] for k in FORMS}
    got = {}
    for rep in range(args.reps + 1):                   # the first round warms every form up
        for name in FORMS:
            h, x, y, cap, w = handles[name]
            check(lib.b200_ars_reset(h), "b200_ars_reset")
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            out = C.c_size_t()
            e0.record()
            check(lib.b200_ars_process(h, x.data_ptr(), n, y.data_ptr(), cap, C.byref(out), None), "b200_ars_process")
            e1.record()
            torch.cuda.synchronize()
            got[name] = out.value
            if rep:
                times[name].append(e0.elapsed_time(e1) * 1e3)
    for name in FORMS:
        h, x, y, cap, w = handles[name]
        us = sorted(times[name])[len(times[name]) // 2]
        nbytes = (n + got[name]) * ch * w
        print(json.dumps({"form": name, "rates": "48000->44100", "channels": ch, "seconds": args.seconds,
                          "us_per_buffer": round(us, 1), "x_realtime": round(args.seconds / (us * 1e-6), 1),
                          "algorithmic_bytes": nbytes, "algorithmic_GB_per_s": round(nbytes / (us * 1e-6) / 1e9, 1),
                          "median_of": args.reps, **dev}))
        lib.b200_ars_destroy(h)


if __name__ == "__main__":
    main()
