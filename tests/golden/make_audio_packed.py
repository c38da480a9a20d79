#!/usr/bin/env python
"""tests/golden/make_audio_packed.py — writes tests/golden/audio_packed.npz and audio_packed_cases.json: audioresample
on every packed sample format as the reference build computes it (oracle/_ref/libgstref_packed.so: unpack, resample,
quantize, pack), so that the oracle and the kernels are pinned where the reference's sources are absent.  Each case is
one stream: two buffers and a drain; the arrays hold each call's input and output bytes.

    python tests/golden/make_audio_packed.py        # rewrite the fixture (needs the reference build)
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ars_packed_cases as pc  # noqa: E402

NPZ, CASES = os.path.join(HERE, "audio_packed.npz"), os.path.join(HERE, "audio_packed_cases.json")
CALLS = [300, 77, None]                 # None: drain, max_latency frames of silence


def cases():
    out = []
    for k, fmt in enumerate(pc.NAMES):
        for o, (a, b, ch, q) in [(pc.OPTS[0], (48000, 44100, 2, 4)), (pc.OPTS[7], (44100, 48001, 3, 4)), (pc.OPTS[10], (3, 2, 2, 5))]:
            out.append({"fmt": fmt, "opts": list(o), "rates": [a, b], "channels": ch, "quality": q, "seed": k})
    return out


def run_ref(c):
    r = pc.ref()
    o, (a, b), ch, fmt = c["opts"], c["rates"], c["channels"], c["fmt"]
    h = r.ref_ars_new_packed(a, b, ch, c["quality"], pc.FORMATS[fmt][0], pc.REF_METHOD[o[0]], pc.REF_MODE[o[1]], pc.REF_INTERP[o[2]])
    rng = np.random.default_rng(c["seed"])
    ins, outs = [], []
    try:
        for n in CALLS:
            x = None if n is None else pc.packed_signal(rng, n, ch, fmt)
            if n is None:
                n = r.ref_ars_max_latency(r.ref_ars_packed_resampler(h))
            cap = int(n * b / a) + 64
            y = np.full(pc.n_bytes(fmt, cap, ch), 7, dtype=np.uint8)
            got = r.ref_ars_process_packed(h, x.ctypes.data if x is not None else None, n, y.ctypes.data, cap)
            ins.append(np.zeros(0, np.uint8) if x is None else x)
            outs.append(y[:pc.n_bytes(fmt, got, ch)])
    finally:
        r.ref_ars_free_packed(h)
    return ins, outs


if __name__ == "__main__":
    assert pc.have_ref(), "needs oracle/_ref/libgstref_packed.so (make -C oracle -f packed.mk)"
    arrays, cs = {}, cases()
    for i, c in enumerate(cs):
        ins, outs = run_ref(c)
        for j, (x, y) in enumerate(zip(ins, outs)):
            arrays["c%d_in%d" % (i, j)], arrays["c%d_out%d" % (i, j)] = x, y
    np.savez_compressed(NPZ, **arrays)
    with open(CASES, "w") as f:
        json.dump({"calls": CALLS, "cases": cs}, f, indent=0)
    print("wrote", NPZ, CASES)
