#!/usr/bin/env python
"""tests/golden/make_vcs_formats.py — writes tests/golden/vcs_formats.json: what the library makes of each video format.

It pins every place a format's facts reach, over all 26 b200_video_format values, so that a change to how the library
describes a format (plane layout, U / V planes, chroma sub-sampling, component bytes, caps defaults) shows up here:

  "info"    b200_video_info_set_format (status and every field) and b200_video_info_size, for every format and a few
            unknown values at INFO_SIZES; b200_video_info_size also for each plane's stride - 1 and offset + 1 / + 2.
  "status"  per "<in>><out>" pair, one character per grid point (STATUS) of b200_vcs_create on a host-only handle
            (device -1).  The grid (points () below) crosses CREATE_SIZES, the default layout and each used plane's
            stride - 1 / offset + 1 / offset + 2 on either side, COLORIMETRY, and no / an odd-origin destination rectangle.
  "plans"   per pair, a digest over the introspection of every accepted grid point: get_plan_info, get_matrix,
            get_chroma_plan, get_taps in both directions and kernel_name.
  "bytes"   per pair accepted at CONVERT_SIZES, a digest of the output frames of emulated converts on a device handle
            (record-only mode off) over CONVERT_SIZES x (no rectangle, a rectangle with each of BORDERS) x (set, zero)
            colorimetry: what introspection cannot see - component byte selectors, de-interleave, border pixel.

It runs the emulated library (tests/cudaemu) like make_vcs_routes.py.

    python tests/golden/make_vcs_formats.py        # rewrite the fixture
"""
import ctypes as C
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "cudaemu"))
FIXTURE = os.path.join(HERE, "vcs_formats.json")

# every b200_video_format of include/b200dsp.h
FMT = {"I420": 2, "YV12": 3, "YUY2": 4, "UYVY": 5, "RGBx": 7, "BGRx": 8, "xRGB": 9, "xBGR": 10, "RGBA": 11, "BGRA": 12,
       "ARGB": 13, "ABGR": 14, "Y42B": 18, "YVYU": 19, "Y444": 20, "NV12": 23, "NV21": 24, "I420_10LE": 43,
       "I422_10LE": 45, "Y444_10LE": 47, "I420_12LE": 73, "I422_12LE": 75, "Y444_12LE": 77, "Y444_16LE": 88,
       "RGBP": 99, "BGRP": 100}
UNKNOWN = [0, 1, 16, 101]
INFO_SIZES = [(1, 1), (2, 2), (33, 17), (64, 48), (720, 577)]
CREATE_SIZES = [(64, 48, 64, 48), (33, 17, 21, 13)]
# set: what b200_video_info_set_format fills in; zero: every colorimetry field left to the library's defaults;
# matrix: an output matrix that differs from the input's; site: an explicit output chroma site
COLORIMETRY = ["set", "zero", "matrix", "site"]
CONVERT_SIZES = [(34, 18, 20, 12), (64, 32, 32, 16)]
BORDERS = [0xff204060, 0x80c0a010]
STATUS = {0: "o", -1: "i", -2: "u", -3: "d", -4: "c", -5: "m", -6: "s"}


def load():
    import build_emu
    from gstreamer_b200 import _lib
    lib = C.CDLL(build_emu.build())
    for name, (res, args) in _lib._SIGS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    lib.b200emu_set_record_only.argtypes = [C.c_int]
    return lib, _lib


def fields(vi):
    return [vi.format, vi.width, vi.height, list(vi.stride), list(vi.offset), vi.color_matrix, vi.color_range,
            vi.chroma_site]


def record_info(lib, c):
    """{format name or number: [[status, fields, size, [size per perturbed layout]] per INFO_SIZES]}"""
    out = {}
    for name in list(FMT) + UNKNOWN:
        rows = []
        for w, h in INFO_SIZES:
            vi = c.VideoInfoC()
            C.memset(C.byref(vi), 0x5A, C.sizeof(vi))
            st = lib.b200_video_info_set_format(C.byref(vi), FMT.get(name, name), w, h)
            sizes = []
            for k in range(4):
                for field, delta in (("stride", -1), ("offset", 1), ("offset", 2)):
                    v2 = c.VideoInfoC.from_buffer_copy(vi)
                    getattr(v2, field)[k] += delta
                    sizes.append(lib.b200_video_info_size(C.byref(v2)))
            rows.append([st, fields(vi), lib.b200_video_info_size(C.byref(vi)), sizes])
        out[str(name)] = rows
    return out


def infos(lib, c, fi, fo, size, colorimetry):
    iw, ih, W, H = size
    ii, oi = c.VideoInfoC(), c.VideoInfoC()
    lib.b200_video_info_set_format(C.byref(ii), FMT[fi], iw, ih)
    lib.b200_video_info_set_format(C.byref(oi), FMT[fo], W, H)
    if colorimetry == "zero":
        for vi in (ii, oi):
            vi.color_matrix = vi.color_range = vi.chroma_site = 0
    elif colorimetry == "matrix":
        oi.color_matrix = 6 if ii.color_matrix != 6 else 3           # BT2020, or BT709 against a BT2020 input
    elif colorimetry == "site":
        oi.chroma_site = 2 | 4                                       # H_COSITED | V_COSITED
    return ii, oi


def layouts(ii, oi):
    """the default layout, then each used plane's stride - 1, offset + 1 and offset + 2, input planes first"""
    yield ii, oi
    for side in (0, 1):
        for k in range(4):
            if (ii, oi)[side].stride[k] == 0:
                continue
            for field, delta in (("stride", -1), ("offset", 1), ("offset", 2)):
                pair = [type(ii).from_buffer_copy(ii), type(oi).from_buffer_copy(oi)]
                getattr(pair[side], field)[k] += delta
                yield pair


def config(c, lib, W, H, dest, border=BORDERS[0]):
    cfg = c.VcsConfigC()
    lib.b200_vcs_config_init(C.byref(cfg))
    if dest:
        cfg.dest_x, cfg.dest_y, cfg.dest_width, cfg.dest_height = 3, 3, W // 2, H // 2
        cfg.border_argb = border
    return cfg


def points(lib, c, fi, fo):
    """(in info, out info, config) of every grid point of a pair, in the fixture's order"""
    for size in CREATE_SIZES:
        for colorimetry in COLORIMETRY:
            ii0, oi0 = infos(lib, c, fi, fo, size, colorimetry)
            for ii, oi in layouts(ii0, oi0):
                for dest in (False, True):
                    yield ii, oi, config(c, lib, size[2], size[3], dest)


def introspect(lib, c, h, hsh, W, H):
    info = c.VcsPlanInfoC()
    hsh.update(b"%d" % lib.b200_vcs_get_plan_info(h, C.byref(info)))
    hsh.update(bytes(info))
    im = (C.c_int32 * 16)()
    hsh.update(b"%d" % lib.b200_vcs_get_matrix(h, im))
    hsh.update(bytes(im))
    cm = (C.c_uint8 * 64)(*([0xEE] * 64))
    hsh.update(b"%d" % lib.b200_vcs_get_chroma_plan(h, cm, 64))
    hsh.update(bytes(cm))
    for d, n in ((0, W), (1, H)):
        offs = (C.c_uint32 * 64)(*([0xFFFFFFFF] * 64))
        taps = (C.c_int16 * 4096)()
        r = lib.b200_vcs_get_taps(h, d, offs, taps, 64, 4096)
        hsh.update(b"%d" % r)
        hsh.update(bytes(offs)[:4 * n])
        if r > 0:
            hsh.update(bytes(taps)[:2 * n * r])
    hsh.update(lib.b200_vcs_kernel_name(h))


def record_pairs(lib, c, fi):
    """({"<fi>><fo>": status string}, {"<fi>><fo>": plan digest}) for every output format"""
    status, plans = {}, {}
    for fo in FMT:
        chars, hsh = [], hashlib.sha256()
        for n, (ii, oi, cfg) in enumerate(points(lib, c, fi, fo)):
            h = C.c_void_p()
            st = lib.b200_vcs_create(C.byref(ii), C.byref(oi), C.byref(cfg), -1, C.byref(h))
            chars.append(STATUS.get(st, "?"))
            if st == 0:
                hsh.update(b"@%d" % n)
                introspect(lib, c, h, hsh, oi.width, oi.height)
                lib.b200_vcs_destroy(h)
        status["%s>%s" % (fi, fo)] = "".join(chars)
        if "o" in chars:
            plans["%s>%s" % (fi, fo)] = hsh.hexdigest()[:32]
    return status, plans


def frame_bytes(n, seed):
    return (C.c_uint8 * n).from_buffer_copy(hashlib.shake_256(seed.encode()).digest(n))


def record_bytes(lib, c, fi):
    """{"<fi>><fo>": output digest} for every output format the default layout accepts at CONVERT_SIZES"""
    lib.b200emu_set_record_only(0)
    out = {}
    for fo in FMT:
        hsh, accepted = hashlib.sha256(), False
        for size in CONVERT_SIZES:
            for colorimetry in ("set", "zero"):
                ii, oi = infos(lib, c, fi, fo, size, colorimetry)
                src = frame_bytes(lib.b200_video_info_size(C.byref(ii)), "%s %dx%d" % (fi, size[0], size[1]))
                for dest, border in [(False, 0)] + [(True, b) for b in BORDERS]:
                    cfg = config(c, lib, size[2], size[3], dest, border)
                    h = C.c_void_p()
                    st = lib.b200_vcs_create(C.byref(ii), C.byref(oi), C.byref(cfg), 0, C.byref(h))
                    hsh.update(b"create %d" % st)
                    if st != 0:
                        continue
                    accepted = True
                    dst = (C.c_uint8 * (lib.b200_video_info_size(C.byref(oi)) + 64))()
                    C.memset(dst, 0x5A, C.sizeof(dst))
                    hsh.update(b"convert %d" % lib.b200_vcs_convert(h, src, dst, None))
                    hsh.update(bytes(dst))
                    lib.b200_vcs_destroy(h)
        if accepted:
            out["%s>%s" % (fi, fo)] = hsh.hexdigest()[:32]
    return out


def record():
    lib, c = load()
    data = {"grid": {"formats": FMT, "unknown": UNKNOWN, "info_sizes": INFO_SIZES, "create_sizes": CREATE_SIZES,
                     "colorimetry": COLORIMETRY, "convert_sizes": CONVERT_SIZES, "borders": BORDERS, "status": STATUS},
            "info": record_info(lib, c), "status": {}, "plans": {}, "bytes": {}}
    for fi in FMT:
        status, plans = record_pairs(lib, c, fi)
        data["status"].update(status)
        data["plans"].update(plans)
        data["bytes"].update(record_bytes(lib, c, fi))
    return data


def write(data, path=FIXTURE):
    with open(path, "w") as f:
        f.write("{\n")
        f.write('"grid": %s,\n' % json.dumps(data["grid"]))
        sections = ["info", "status", "plans", "bytes"]
        for i, s in enumerate(sections):
            f.write('"%s": {\n' % s + ",\n".join("%s: %s" % (json.dumps(k), json.dumps(v)) for k, v in data[s].items()))
            f.write("\n}" + (",\n" if i < len(sections) - 1 else "\n"))
        f.write("}\n")


if __name__ == "__main__":
    write(record(), sys.argv[1] if len(sys.argv) > 1 else FIXTURE)
