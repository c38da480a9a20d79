#!/usr/bin/env python
"""tests/golden/make_ars_packed_routes.py — writes tests/golden/ars_packed_routes.json: the kernels a b200_ars handle
launches for each way a packed sample format is stored (tests/ars_packed_cases.py CLASSES), over the option sets and rate
pairs that reach the direct kernel in FULL and interpolated mode, the small kernel and the equal-rate copy.  Recorded
with make_ars_routes.Recorder (the emulated library in record-only mode) with the same call sequence, the pointers at
odd byte offsets instead of below 16-byte alignment.

    python tests/golden/make_ars_packed_routes.py        # rewrite the fixture
"""
import ctypes as C
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
FIXTURE = os.path.join(HERE, "ars_packed_routes.json")

import ars_packed_cases as pc  # noqa: E402
import make_ars_routes as mr  # noqa: E402

OPTS = [pc.OPTS[0], pc.OPTS[3], pc.OPTS[7], pc.OPTS[9], pc.OPTS[11]]
RATES = [(48000, 44100, 4), mr.INTERP_PAIR, (44100, 44100, 4), (3, 2, 4)]
SEQ = [(1, 16), (2000, 16), (None, 16), (480, 1), (480, 3)], [(300, 16)]


def grid():
    for fmt in pc.CLASSES:
        for o in OPTS:
            for r in RATES:
                yield "%s %s %d>%d q%d" % (fmt, "-".join(o), *r), fmt, o, r


def record():
    rec = mr.Recorder()
    out = {}
    try:
        for key, fmt, o, (a, b, q) in grid():
            cfg = pc.config(None, a, b, 2, q, fmt, o)
            h = C.c_void_p()
            st = rec.lib.b200_ars_create(C.byref(cfg), 0, C.byref(h))
            if st != 0:
                out[key] = [st]
                continue
            try:
                row = [st, rec.plan_info(h), rec.run(h, SEQ[0])]
                assert rec.lib.b200_ars_update(h, *mr.update_rates((a, b))) == 0
                out[key] = row + [rec.plan_info(h), rec.run(h, SEQ[1])]
            finally:
                rec.lib.b200_ars_destroy(h)
    finally:
        rec.lib.b200emu_set_record_only(0)
        rec.lib.b200emu_clear_launch_log()
    return out


if __name__ == "__main__":
    with open(FIXTURE, "w") as f:
        json.dump(record(), f, indent=0, sort_keys=True)
    print("wrote", FIXTURE)
