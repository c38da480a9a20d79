#!/usr/bin/env python
"""Generates tests/golden/video_rgbp.npz + video_rgbp_cases.json from the reference's OWN code (oracle/_ref/libgstref.so,
built by oracle/Makefile from the reference sources): planar RGB outputs (RGBP / BGRP) of 4:2:0, packed 4:2:2, planar
4:4:4 and packed RGB inputs, I420 at an unchanged size included (no convert_I420_BGRA-style row for planar outputs).
Run in the build container only:

    python tests/golden/make_golden_rgbp.py

Inputs are regenerated from seeds (numpy default_rng over the input frame's size), so only seeds, parameters and the
reference's output bytes are stored; output frames have the default layout (three planes of stride ROUND_UP_4 (w))."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import bindings as ob  # noqa: E402
from rgbp_oracle import FMT, default_layout, frame_size  # noqa: E402


def video_rgbp():
    arrays, cases = {}, []
    for fi, fo in [("NV12", "RGBP"), ("I420", "BGRP"), ("YV12", "RGBP"), ("NV21", "BGRP"), ("YUY2", "RGBP"), ("Y444", "BGRP"),
                   ("BGRA", "RGBP"), ("xRGB", "BGRP")]:
        for (iw, ih, ow, oh) in [(64, 48, 32, 24), (40, 30, 52, 39), (65, 49, 33, 25), (33, 17, 20, 31), (50, 21, 50, 21), (1, 1, 1, 1)]:
            for m, site in ((1, 2), (3, 1), (9, 2)):
                d = ob.vcs_desc(iw, ih, iw, ih, m, in_fmt=FMT[fi], out_fmt=FMT["BGRx"])
                frame = np.random.default_rng(m + iw).integers(0, 256, ob.vcs_sizes(d)[0], dtype=np.uint8)
                rgb_in = fi in ("BGRA", "xRGB")
                r = ob.RefVcs(iw, ih, ow, oh, m, in_fmt=FMT[fi], out_fmt=FMT[fo], site=-1 if rgb_in else site)
                out = r.convert(frame, np.zeros(frame_size(default_layout(ow, oh), oh), dtype=np.uint8))
                r.close()
                key = f"g_{fi}_{fo}_{iw}x{ih}_{ow}x{oh}_m{m}"
                arrays[key] = out
                cases.append({"key": key, "in_fmt": fi, "out_fmt": fo, "in": [iw, ih], "out": [ow, oh], "method": m,
                              "site": None if rgb_in else site, "seed": m + iw})
    np.savez_compressed(os.path.join(HERE, "video_rgbp.npz"), **arrays)
    json.dump(cases, open(os.path.join(HERE, "video_rgbp_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    assert ob.have_ref(), "needs oracle/_ref/libgstref.so (make -C oracle ref)"
    video_rgbp()
    print("golden fixtures written to", HERE)
