#!/usr/bin/env python
"""tests/golden/make_vcs_geometry.py — writes tests/golden/vcs_geometry.json: the launch geometry of every tiled kernel.

Each record is one device handle and one convert of 16-byte aligned frames: the create status, get_plan_info's tile_w,
tile_h and smem_bytes (the generic kernel's tile), the convert status and its launches, each with its grid, block and
dynamic shared-memory bytes.  The tile shapes, staged extents and shared-memory sizes of the generic, light, n-tap and
plane kernels all show in those numbers.  The grids: make_vcs_routes' main grid (every format pair, chroma siting,
size, method and destination rectangle), then production sizes for every method over pairs that reach the generic,
light, n-tap and plane kernels and the packed RGB -> 4:2:0 and RGBP scalers (PROD).  Each tile-shape override (KNOBS)
is recorded over PROD in a process of its own, set to a shape the search would not pick.  It runs the emulated library
(tests/cudaemu) in record-only mode: every launch is logged, no block runs.

Layout: "cases" maps "<in>><out>" to a digest of that pair's records over the main grid, "prod" the same over PROD,
"knobs" the same over PROD per knob.  A digest is the first 16 hex digits of the SHA-256 of the JSON list of
[key, record] in grid () order; a record is [create status] or [0, tile_w, tile_h, smem_bytes, convert status,
launches].  `--dump PAIR` prints one pair's records of the main grid, to see what changed.

    python tests/golden/make_vcs_geometry.py        # rewrite the fixture
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_vcs_routes as mr  # noqa: E402

FIXTURE = os.path.join(HERE, "vcs_geometry.json")
MAIN = {"pairs": mr.MAIN_GRID["pairs"], "sizes": mr.SIZES, "dests": (False, True)}
PROD = {"pairs": [("NV12", "BGRA"), ("I420", "BGRA"), ("NV12", "NV12"), ("I420", "I420"), ("BGRA", "BGRA"), ("BGRA", "NV12"),
                  ("BGRA", "RGBP")],
        "sizes": [(3840, 2160, 1920, 1080), (1920, 1080, 1280, 720), (1280, 720, 1920, 1080), (1920, 1080, 640, 640),
                  (1917, 1079, 853, 479)],
        "dests": (False,)}
# tile overrides, each a shape the search does not pick for any PROD case
KNOBS = ["B200_NTAP_SHAPE=64,8", "B200_PLF_SHAPE=32,8", "B200_LIGHT_TH=4"]
FRAME = 3840 * 2160 * 4 + (1 << 16)                        # the largest frame of the grids, with room for the offsets


class Recorder:
    def __init__(self):
        self.lib, self.c = mr.load()
        self.lib.b200emu_set_record_only(2)
        self.buf = (C.c_uint8 * (2 * FRAME + 64))()
        self.base = (C.addressof(self.buf) + 63) & ~63

    def handle(self, fi, fo, site, size, dest, method):
        iw, ih, W, H = size
        lib, c = self.lib, self.c
        ii, oi = c.VideoInfoC(), c.VideoInfoC()
        assert lib.b200_video_info_set_format(C.byref(ii), mr.FMT[fi], iw, ih) == 0
        assert lib.b200_video_info_set_format(C.byref(oi), mr.FMT[fo], W, H) == 0
        if site is not None:
            ii.chroma_site = site
        if fi in mr.YUV420 and fo in mr.YUV420:            # what the element's caps fixation does
            oi.color_matrix, oi.color_range, oi.chroma_site = ii.color_matrix, ii.color_range, ii.chroma_site
        cfg = c.VcsConfigC()
        lib.b200_vcs_config_init(C.byref(cfg))
        cfg.method = method
        if dest:
            cfg.dest_x, cfg.dest_y, cfg.dest_width, cfg.dest_height = mr.dest_rect(W, H)
            cfg.border_argb = 0xff204060
        h = C.c_void_p()
        st = lib.b200_vcs_create(C.byref(ii), C.byref(oi), C.byref(cfg), 0, C.byref(h))
        if st != 0:
            return [st]
        try:
            info = c.VcsPlanInfoC()
            assert lib.b200_vcs_get_plan_info(h, C.byref(info)) == 0
            lib.b200emu_clear_launch_log()
            cst = lib.b200_vcs_convert(h, self.base, self.base + FRAME, None)
            log = lib.b200emu_launch_log().decode()
            lib.b200emu_clear_launch_log()
            return [st, info.tile_w, info.tile_h, info.smem_bytes, cst, [x for x in log.split("\n") if x]]
        finally:
            lib.b200_vcs_destroy(h)


def grid(pairs, sizes, dests):
    """(key, in, out, site, size, dest, method) of every record, in the fixture's order"""
    for fi, fo in pairs:
        for site in mr.SITES if fi not in mr.RGB else [None]:
            for size in sizes:
                for dest in dests:
                    for m in mr.METHODS:
                        key = "%s>%s %s %dx%d>%dx%d %s m%d" % (fi, fo, "site-" if site is None else "site%d" % site, *size,
                                                              "dest" if dest else "full", m)
                        yield key, fi, fo, site, size, dest, m


def record_rows(g):
    """[(key, record)] of grid g, from the library the emulator builds from gstreamer_b200/csrc"""
    rec = Recorder()
    try:
        return [(key, rec.handle(*args)) for key, *args in grid(**g)]
    finally:                                               # the library is shared with the other tests of the process
        rec.lib.b200emu_set_record_only(0)
        rec.lib.b200emu_clear_launch_log()


def record_knob(knob):
    """record_rows of PROD in a process of its own with the environment variable `knob` ("NAME=value") set"""
    name, value = knob.split("=")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--knob-rows"], env={**os.environ, name: value},
                       capture_output=True, text=True, check=True)
    return json.loads(r.stdout)


def digests(rows):
    """{"<in>><out>": digest of that pair's [key, record] list}"""
    pairs = {}
    for key, r in rows:
        pairs.setdefault(key.split()[0], []).append([key, r])
    return {p: hashlib.sha256(json.dumps(v).encode()).hexdigest()[:16] for p, v in pairs.items()}


def record():
    """the fixture's content"""
    return {"grid": {"main": MAIN, "prod": PROD, "sites": mr.SITES, "methods": len(mr.METHODS)},
            "cases": digests(record_rows(MAIN)), "prod": digests(record_rows(PROD)),
            "knobs": {k: digests(record_knob(k)) for k in KNOBS}}


def write(data, path=FIXTURE):
    by_input = {}
    for pair, d in data["cases"].items():
        by_input.setdefault(pair.split(">")[0], []).append(json.dumps({pair: d})[1:-1])
    with open(path, "w") as f:
        f.write('{\n"grid": %s,\n' % json.dumps(data["grid"]))
        f.write('"cases": {\n' + ",\n".join(", ".join(v) for v in by_input.values()) + "\n},\n")
        f.write('"prod": %s,\n' % json.dumps(data["prod"]))
        f.write('"knobs": {\n' + ",\n".join("%s: %s" % (json.dumps(k), json.dumps(v)) for k, v in data["knobs"].items()) + "\n}\n}\n")


if __name__ == "__main__":
    if sys.argv[1:] == ["--knob-rows"]:
        json.dump(record_rows(PROD), sys.stdout)
    elif sys.argv[1:2] == ["--dump"]:
        g = dict(MAIN, pairs=[tuple(sys.argv[2].split(">"))])
        for key, r in record_rows(g):
            print(key, json.dumps(r))
    else:
        write(record(), sys.argv[1] if len(sys.argv) > 1 else FIXTURE)
