#!/usr/bin/env python
"""tests/golden/make_vcs_routes.py — writes tests/golden/vcs_routes.json: which kernels a b200_vcs handle launches.

For every sink x source format pair cudavideoconvertscale accepts, the input's default and h-cosited chroma siting (YUV
inputs; the 2:1 kernel needs the latter), sizes that reach every route, all ten methods, with and without a bordered
destination rectangle, it records what the library reports for the default kernel and for each forced variant (create
and set_kernel_variant status, plan_info kernel_variant and n_launches_per_convert, kernel_name) and, for device
handles, the status and the kernels of one convert with in / out frames at 16-, 8-, 4- and 1-byte alignment.  Host-only
handles (device -1) record the introspection only.  Each A/B knob (KNOBS) is recorded over a smaller grid in a process
of its own with the knob set.  It runs the emulated library (tests/cudaemu) in record-only mode: every launch is logged,
no block runs.  The wgmma variant (7) is not emulated.

Layout: "launches" lists the distinct launch sequences, "results" the distinct per-handle records, "rows" the distinct
lists of one result index per method (0..9).  "cases" maps "<in>><out>" to one row index per site x size x (full,
dest) x (device 0, host-only), in that order (grid () below; expand () gives every record under its own key);
"knobs" does the same per knob over KNOB_GRID.  A result is [create status, state...]; a state is [forced variant or
null, set status, kernel_variant, n_launches_per_convert, kernel_name, converts or null], converts one [status,
launches index] per alignment.  The variants are forced one after another on the same handle: a refused one leaves the
previous in place.

    python tests/golden/make_vcs_routes.py        # rewrite the fixture
"""
import ctypes as C
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "cudaemu"))
FIXTURE = os.path.join(HERE, "vcs_routes.json")

# the element's caps (gst/gstcudavideoconvertscale.c SINK_FORMATS / SRC_FORMATS), b200_video_format values
FMT = {"NV12": 23, "NV21": 24, "I420": 2, "YV12": 3, "BGRA": 12, "RGBA": 11, "ARGB": 13, "ABGR": 14, "BGRx": 8,
       "RGBx": 7, "xRGB": 9, "xBGR": 10, "YUY2": 4, "UYVY": 5, "YVYU": 19, "Y42B": 18, "Y444": 20, "RGBP": 99, "BGRP": 100}
YUV420 = ["NV12", "NV21", "I420", "YV12"]
RGB = ["BGRA", "RGBA", "ARGB", "ABGR", "BGRx", "RGBx", "xRGB", "xBGR"]
SINKS = YUV420 + RGB + ["YUY2", "UYVY", "YVYU", "Y42B", "Y444"]
SRCS = RGB + ["RGBP", "BGRP"] + YUV420
SIZES = [
    (64, 48, 64, 48),     # unchanged
    (128, 64, 64, 32),    # exact 2:1, output width a multiple of 16
    (72, 40, 36, 20),     # exact 2:1, other widths
    (100, 60, 64, 36),    # down-scale
    (40, 30, 64, 48),     # up-scale
    (33, 17, 21, 13),     # odd width and height
    (35, 17, 35, 17),     # odd, unchanged
    (64, 48, 64, 30),     # vertical only
    (64, 48, 40, 48),     # horizontal only
    (64, 1, 40, 1),       # one line
]
# the input's chroma siting: the default of its size (none at these sizes), and h-cosited, which the 2:1 kernel needs
SITES = [None, 2]
METHODS = range(10)
VARIANTS = [0, 1, 2, 3, 6]
ALIGNS = [16, 8, 4, 1]
MAIN_GRID = {"pairs": [(fi, fo) for fi in SINKS for fo in SRCS]}
# the A/B knobs, each set for the whole of a smaller grid: pairs and sizes the knobs act on
KNOBS = ["B200_CROSS_GENERIC=1", "B200_RGB420_GENERIC=1", "B200_L2_V1=1", "B200_L2_X4=0", "B200_PLANES_SLOW=1"]
KNOB_GRID = {"pairs": [("NV12", "BGRA"), ("I420", "RGBA"), ("NV12", "RGBP"), ("NV12", "I420"), ("I420", "NV12"), ("NV12", "NV12"),
                       ("I420", "I420"), ("BGRA", "NV12"), ("BGRA", "RGBP"), ("YUY2", "I420"), ("UYVY", "NV12")],
             "sizes": [(128, 64, 64, 32), (100, 60, 64, 36), (35, 17, 35, 17), (40, 30, 64, 48)], "dests": (False,)}


def load():
    import build_emu
    from gstreamer_b200 import _lib
    lib = C.CDLL(build_emu.build())
    for name, (res, args) in _lib._SIGS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    lib.b200emu_launch_log.restype = C.c_char_p
    lib.b200emu_set_record_only.argtypes = [C.c_int]
    return lib, _lib


def dest_rect(W, H):
    return (2, 2, W - 4, H - 4) if H > 4 else (2, 0, W - 4, H)


class Recorder:
    def __init__(self):
        self.lib, self.c = load()
        self.lib.b200emu_set_record_only(1)
        self.buf = (C.c_uint8 * (1 << 20))()
        base = C.addressof(self.buf)
        self.base = (base + 63) & ~63                      # 64-byte aligned: offset k gives alignment min(16, k & -k)

    def launches(self):
        log = self.lib.b200emu_launch_log().decode()
        self.lib.b200emu_clear_launch_log()
        return [x for x in log.split("\n") if x]

    def state(self, h, variant, set_st, device):
        info = self.c.VcsPlanInfoC()
        assert self.lib.b200_vcs_get_plan_info(h, C.byref(info)) == 0
        name = self.lib.b200_vcs_kernel_name(h).decode()
        conv = None
        if device >= 0 and set_st == 0:
            conv = []
            for a in ALIGNS:
                off = 0 if a == 16 else a
                self.lib.b200emu_clear_launch_log()
                st = self.lib.b200_vcs_convert(h, self.base + off, self.base + (1 << 19) + off, None)
                conv.append((st, self.launches()))
        return [variant, set_st, info.kernel_variant, info.n_launches_per_convert, name, conv]

    def handle(self, fi, fo, site, size, method, dest, device):
        iw, ih, W, H = size
        lib, c = self.lib, self.c
        ii, oi = c.VideoInfoC(), c.VideoInfoC()
        assert lib.b200_video_info_set_format(C.byref(ii), FMT[fi], iw, ih) == 0
        assert lib.b200_video_info_set_format(C.byref(oi), FMT[fo], W, H) == 0
        if site is not None:
            ii.chroma_site = site
        if fi in YUV420 and fo in YUV420:                  # what the element's caps fixation does
            oi.color_matrix, oi.color_range, oi.chroma_site = ii.color_matrix, ii.color_range, ii.chroma_site
        cfg = c.VcsConfigC()
        lib.b200_vcs_config_init(C.byref(cfg))
        cfg.method = method
        if dest:
            cfg.dest_x, cfg.dest_y, cfg.dest_width, cfg.dest_height = dest_rect(W, H)
            cfg.border_argb = 0xff204060
        h = C.c_void_p()
        st = lib.b200_vcs_create(C.byref(ii), C.byref(oi), C.byref(cfg), device, C.byref(h))
        if st != 0:
            return [st]
        try:
            out = [st, self.state(h, None, 0, device)]
            for v in VARIANTS:
                s = lib.b200_vcs_set_kernel_variant(h, v)
                out.append(self.state(h, v, s, device))
        finally:
            lib.b200_vcs_destroy(h)
        return out


def grid(pairs, sizes=SIZES, dests=(False, True)):
    """(key, in, out, site, size, dest, device) of every row, in the fixture's order"""
    for fi, fo in pairs:
        for site in SITES if fi not in RGB else [None]:
            for size in sizes:
                for dest in dests:
                    for device in (0, -1):
                        key = "%s>%s %s %dx%d>%dx%d %s %s" % (fi, fo, "site-" if site is None else "site%d" % site, *size,
                                                             "dest" if dest else "full", "dev" if device >= 0 else "host")
                        yield key, fi, fo, site, size, dest, device


def record_rows(gridargs):
    """[(key, [result per method])] with launch lists, from the library the emulator builds from gstreamer_b200/csrc"""
    rec = Recorder()
    out = []
    try:
        for key, fi, fo, site, size, dest, device in grid(**gridargs):
            out.append((key, [rec.handle(fi, fo, site, size, m, dest, device) for m in METHODS]))
    finally:                                               # the library is shared with the other tests of the process
        rec.lib.b200emu_set_record_only(0)
        rec.lib.b200emu_clear_launch_log()
    return out


def record_knob(knob):
    """record_rows of the knob grid in a process of its own with the environment variable `knob` ("NAME=value") set"""
    name, value = knob.split("=")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--knob-rows"], env={**os.environ, name: value},
                       capture_output=True, text=True, check=True)
    return json.loads(r.stdout)


def record():
    """the fixture's content"""
    tables = {"launches": [], "results": [], "rows": []}
    index = {t: {} for t in tables}

    def intern(table, v):
        k = json.dumps(v)
        if k not in index[table]:
            index[table][k] = len(tables[table])
            tables[table].append(v)
        return index[table][k]

    def cases(rows):
        out = {}
        for key, results in rows:
            for r in results:
                for s in r[1:]:
                    if s[5] is not None:
                        s[5] = [[st, intern("launches", l)] for st, l in s[5]]
            out.setdefault(key.split()[0], []).append(intern("rows", [intern("results", r) for r in results]))
        return out

    main = cases(record_rows(MAIN_GRID))
    knobs = {k: cases(record_knob(k)) for k in KNOBS}
    return {"grid": {"sizes": SIZES, "sites": SITES, "dest": [False, True], "device": [0, -1], "methods": len(METHODS),
                     "variants": VARIANTS, "aligns": ALIGNS, "knob_pairs": KNOB_GRID["pairs"], "knob_sizes": KNOB_GRID["sizes"]},
            **tables, "cases": main, "knobs": knobs}


def expand(data, knob=None):
    """{row key: [result per method]} of the main grid (or of one knob's grid), launch indices replaced by the lists"""
    cases, gridargs = (data["cases"], MAIN_GRID) if knob is None else (data["knobs"][knob], KNOB_GRID)
    out = {}
    it = grid(**gridargs)
    for pair in cases:
        for row in cases[pair]:
            key = next(it)[0]
            res = []
            for ri in data["rows"][row]:
                r = json.loads(json.dumps(data["results"][ri]))
                for s in r[1:]:
                    if s[5] is not None:
                        s[5] = [[st, data["launches"][l]] for st, l in s[5]]
                res.append(r)
            out[key] = res
    return out


def write(data, path=FIXTURE):
    with open(path, "w") as f:
        f.write("{\n")
        f.write('"grid": %s,\n' % json.dumps(data["grid"]))
        for t in ("launches", "results", "rows"):
            f.write('"%s": [\n' % t + ",\n".join(json.dumps(s) for s in data[t]) + "\n],\n")
        f.write('"cases": {\n' + ",\n".join("%s: %s" % (json.dumps(k), json.dumps(v)) for k, v in data["cases"].items()) + "\n},\n")
        f.write('"knobs": {\n' + ",\n".join("%s: %s" % (json.dumps(k), json.dumps(v)) for k, v in data["knobs"].items()) + "\n}\n")
        f.write("}\n")


if __name__ == "__main__":
    if sys.argv[1:] == ["--knob-rows"]:
        json.dump(record_rows(KNOB_GRID), sys.stdout)
    else:
        write(record(), sys.argv[1] if len(sys.argv) > 1 else FIXTURE)
