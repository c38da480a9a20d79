#!/usr/bin/env python
"""tests/golden/make_ars_routes.py — writes tests/golden/ars_routes.json: which kernels a b200_ars handle launches.

A record holds the create status, the plan_info fields and, on one device handle, a short sequence of calls (calls ()):
each call's status, out_frames and launches, every launch with its grid, block and dynamic shared-memory bytes.  The
sequence has a call that yields no output, several buffer sizes, a silent call (no input), input / output pointers below
16-byte alignment, and b200_ars_update to another rate pair (update_rates ()) followed by one more call.

MAIN is a union of grids, each over what changes the route, for every sample format: every resample-method /
sinc-filter-mode / sinc-filter-interpolation set of the emulated kernel tests (OPTS) at 48k -> 44.1k and at the
interpolated-mode pair 44.1k -> 48001; the default and the nearest / linear / cubic methods at equal rates (a copy plan)
and at 3 -> 2 (3 and 12 taps); the default options at 44.1k -> 48k, 48k -> 8k, 96k -> 8k at quality 7 (1480 taps: more
than the tile kernel takes) and 192k -> 4k at quality 10 (12288 taps: refused in F32 FULL mode); then F32 and S16 across
the warp / channel block / whole-128-block boundaries.  Each audio knob (KNOBS) is recorded over KNOB in a process of
its own with the knob set.  B200_ARS_NO_TENSORMAP is not recorded: under emulation the tensor-map encoder is a stub that
always declines, so the knob has nothing to change.  It runs the emulated library (tests/cudaemu) in record-only mode:
every launch is logged, no block runs.  Recording takes about 6 s, tests/test_ars_routes.py about 11 s.

Layout: "launches" lists the distinct launches ("kernel grid=x,y,z block=x,y,z smem=bytes"), "calls" the distinct calls,
"results" the distinct records.  "main" holds one result index per record of grid (MAIN), "knobs" the same per knob over
grid (KNOB); expand () gives every record under its own key.  A result is [create status] or [0, plan_info, call indices,
plan_info after the update, call indices after the update]; plan_info is [n_taps, n_phases, in_step, out_step,
filter_mode, oversample], a call [status, out_frames, launch indices].

    python tests/golden/make_ars_routes.py        # rewrite the fixture
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
FIXTURE = os.path.join(HERE, "ars_routes.json")

# b200_audio_format values
FMT = {"F32": 28, "S16": 4, "S32": 12, "F64": 30}
# tests/test_emu_kernels.py AUDIO_OPTS, in the element's property names
OPTS = [("kaiser", "auto", "cubic"), ("blackman-nuttall", "auto", "cubic"), ("kaiser", "full", "none"),
        ("kaiser", "interpolated", "cubic"), ("blackman-nuttall", "full", "none"), ("kaiser", "interpolated", "none"),
        ("kaiser", "full", "linear"), ("kaiser", "interpolated", "linear"), ("blackman-nuttall", "interpolated", "linear"),
        ("nearest", "auto", "cubic"), ("linear", "auto", "cubic"), ("cubic", "auto", "cubic")]
METHOD = {"nearest": 1, "linear": 2, "cubic": 3, "blackman-nuttall": 4, "kaiser": 5}
MODE = {"interpolated": 1, "full": 2, "auto": 3}
INTERP = {"none": 1, "linear": 2, "cubic": 3}
# (in rate, out rate, quality).  44.1k -> 48001 has 48001 phases: interpolated under "auto"; with "full" forced its table
# would take hundreds of MB, so that pair is left out of the forced-full options.
INTERP_PAIR = (44100, 48001, 4)
MAIN = [{"fmts": list(FMT), "opts": OPTS, "rates": [(48000, 44100, 4), INTERP_PAIR], "channels": [2]},
        {"fmts": list(FMT), "opts": OPTS[:1] + OPTS[9:], "rates": [(44100, 44100, 4), (3, 2, 4)], "channels": [2]},
        {"fmts": list(FMT), "opts": OPTS[:1], "rates": [(44100, 48000, 4), (48000, 8000, 4), (96000, 8000, 7), (192000, 4000, 10)],
         "channels": [2]},
        {"fmts": ["F32", "S16"], "opts": OPTS[:1], "rates": [(48000, 44100, 4), (44100, 48000, 4), (96000, 8000, 7)],
         "channels": [1, 40, 64, 66, 128, 256]}]
IN_FRAMES, OUT_FRAMES = 8000, 16384                  # the largest call and the output capacity
# the pointer alignments below 16 bytes each format's calls use
ALIGNS = {"F32": [8, 4], "S16": [2], "S32": [4], "F64": [8]}
KNOBS = ["B200_ARS_GENERIC=1", "B200_ARS_NOPIPE=1", "B200_ARS_PIPE_V1=1", "B200_ARS_GRID=2", "B200_ARS_NO=16", "B200_ARS_NO=64",
         "B200_ARS_CB=32", "B200_ARS_CB=64", "B200_ARS_CPT=1", "B200_ARS_CPT=4"]
# first: routes no knob may change (equal rates: a copy plan; the interpolated pair); then the F32 / S16 FULL routes
KNOB = [{"fmts": ["F32", "S16"], "opts": OPTS[:1], "rates": [(44100, 44100, 4), INTERP_PAIR], "channels": [2]},
        {"fmts": ["F32", "S16"], "opts": OPTS[:1], "rates": [(48000, 44100, 4), (96000, 8000, 7)], "channels": [2, 40, 66, 128]}]


def calls(fmt):
    """(input frames or None for a silent call of 200 frames, pointer alignment) of the calls before and after the update;
    the first call leaves the history short of one window: no output; the second fills one of 12288 taps"""
    return [(1, 16), (IN_FRAMES, 16), (None, 16)] + [(480, a) for a in ALIGNS[fmt]], [(300, 16)]


def update_rates(rates):
    return (44100, 48000) if rates[:2] == (48000, 44100) else (48000, 44100)


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


class Recorder:
    def __init__(self):
        self.lib, self.c = load()
        self.lib.b200emu_set_record_only(2)
        self.size = 8 * 256 * IN_FRAMES                      # the largest input, F64 x 256 channels; the output follows
        self.buf = (C.c_uint8 * (self.size + 8 * 256 * OUT_FRAMES + 64))()
        self.base = (C.addressof(self.buf) + 63) & ~63       # offset k gives alignment min(16, k & -k)

    def launches(self):
        log = self.lib.b200emu_launch_log().decode()
        self.lib.b200emu_clear_launch_log()
        return [x for x in log.split("\n") if x]

    def plan_info(self, h):
        i = self.c.ArsPlanInfoC()
        assert self.lib.b200_ars_get_plan_info(h, C.byref(i)) == 0
        return [i.n_taps, i.n_phases, i.in_step, i.out_step, i.filter_mode, i.oversample]

    def run(self, h, seq):
        out = []
        for n, align in seq:
            off = 0 if align == 16 else align
            src = None if n is None else self.base + off
            n = 200 if n is None else n
            got = C.c_size_t(12345)
            self.lib.b200emu_clear_launch_log()
            st = self.lib.b200_ars_process(h, src, n, self.base + self.size + off, OUT_FRAMES, C.byref(got), None)
            out.append([st, got.value, self.launches()])
        return out

    def handle(self, fmt, opts, rates, ch):
        cfg = self.c.ArsConfigC()
        cfg.in_rate, cfg.out_rate, cfg.quality = rates
        cfg.channels, cfg.format = ch, FMT[fmt]
        cfg.resample_method, cfg.sinc_filter_mode, cfg.sinc_filter_interpolation = METHOD[opts[0]], MODE[opts[1]], INTERP[opts[2]]
        h = C.c_void_p()
        st = self.lib.b200_ars_create(C.byref(cfg), 0, C.byref(h))
        if st != 0:
            return [st]
        try:
            before, after = calls(fmt)
            out = [st, self.plan_info(h), self.run(h, before)]
            assert self.lib.b200_ars_update(h, *update_rates(rates)) == 0
            out += [self.plan_info(h), self.run(h, after)]
        finally:
            self.lib.b200_ars_destroy(h)
        return out


def grid(grids):
    """(record key, format, options, rate pair, channels) of every record, in the fixture's order"""
    for g in grids:
        for fmt in g["fmts"]:
            for o in g["opts"]:
                for r in g["rates"]:
                    if o[1] == "full" and r == INTERP_PAIR:
                        continue
                    for ch in g["channels"]:
                        yield "%s %s %d>%d q%d %dch" % (fmt, "-".join(o), *r, ch), fmt, o, r, ch


def record_rows(grids):
    """[result] of every record, with launch lists, from the library the emulator builds from gstreamer_b200/csrc"""
    rec = Recorder()
    try:
        return [rec.handle(fmt, o, r, ch) for _, fmt, o, r, ch in grid(grids)]
    finally:                                               # the library is shared with the other tests of the process
        rec.lib.b200emu_set_record_only(0)
        rec.lib.b200emu_clear_launch_log()


def record_knob(knob):
    """record_rows of KNOB in a process of its own with the environment variable `knob` ("NAME=value") set"""
    name, value = knob.split("=")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--knob-rows"], env={**os.environ, name: value},
                       capture_output=True, text=True, check=True)
    return json.loads(r.stdout)


def record():
    """the fixture's content"""
    tables = {"launches": [], "calls": [], "results": []}
    index = {t: {} for t in tables}

    def intern(table, v):
        k = json.dumps(v)
        if k not in index[table]:
            index[table][k] = len(tables[table])
            tables[table].append(v)
        return index[table][k]

    def results(rows):
        for r in rows:
            for i in range(2, len(r), 2):
                r[i] = [intern("calls", [st, n, [intern("launches", x) for x in l]]) for st, n, l in r[i]]
        return [intern("results", r) for r in rows]

    main = results(record_rows(MAIN))
    knobs = {k: results(record_knob(k)) for k in KNOBS}
    return {"grid": {"main": MAIN, "knob": KNOB, "aligns": ALIGNS}, **tables, "main": main, "knobs": knobs}


def expand(data, knob=None):
    """{record key: result} of MAIN (or of KNOB under one knob), call and launch indices replaced by their values"""
    indices, grids = (data["main"], MAIN) if knob is None else (data["knobs"][knob], KNOB)
    keys = [key for key, *_ in grid(grids)]
    assert len(keys) == len(indices)
    out = {}
    for key, ri in zip(keys, indices):
        res = json.loads(json.dumps(data["results"][ri]))
        for i in range(2, len(res), 2):
            res[i] = [[st, n, [data["launches"][x] for x in l]] for st, n, l in (data["calls"][c] for c in res[i])]
        out[key] = res
    return out


def write(data, path=FIXTURE):
    rows = lambda v: ",\n".join(json.dumps(v[i:i + 40])[1:-1] for i in range(0, len(v), 40))   # noqa: E731
    with open(path, "w") as f:
        f.write("{\n")
        f.write('"grid": %s,\n' % json.dumps(data["grid"]))
        for t in ("launches", "calls", "results"):
            f.write('"%s": [\n' % t + ",\n".join(json.dumps(s) for s in data[t]) + "\n],\n")
        f.write('"main": [\n%s\n],\n' % rows(data["main"]))
        f.write('"knobs": {\n' + ",\n".join('%s: [\n%s\n]' % (json.dumps(k), rows(v)) for k, v in data["knobs"].items()) + "\n}\n")
        f.write("}\n")


if __name__ == "__main__":
    if sys.argv[1:] == ["--knob-rows"]:
        json.dump(record_rows(KNOB), sys.stdout)
    else:
        write(record(), sys.argv[1] if len(sys.argv) > 1 else FIXTURE)
