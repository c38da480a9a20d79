"""cudaaudioresample on the sample formats it unpacks (every interleaved GstAudioFormat but S16LE, S32LE, F32LE, F64LE),
without a GPU: the oracle (unpack, resample in S32 / F64, quantize, pack) against the reference's own converter steps,
the golden fixture, the host plan, the launches per format class, and the product's kernels under emulation
(tests/cudaemu) byte for byte against the oracle — streams, drain, reset, rate updates and the system-memory path."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "cudaemu"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import ars_packed_cases as pc  # noqa: E402

pytestmark = pytest.mark.timeout(900)
need_ref = pytest.mark.skipif(not pc.have_ref(), reason="reference build (oracle/_ref/libgstref_packed.so) not present")

# (in rate, out rate, channels, quality): FULL (48k -> 44.1k), interpolated (44.1k -> 48001), the small-method plans
# (3 -> 2: 3 and 12 taps) and the equal-rate copy
RATES = [(48000, 44100, 2, 4), (44100, 48001, 3, 4)]
SMALL_RATES = [(3, 2, 3, 5), (44100, 44100, 2, 4)]


def rates_for(opts):
    return RATES + (SMALL_RATES if pc.REF_METHOD[opts[0]] < 3 else [])


def ref_stream(a, b, ch, q, fmt, opts):
    r = pc.ref()
    h = r.ref_ars_new_packed(a, b, ch, q, pc.FORMATS[fmt][0], pc.REF_METHOD[opts[0]], pc.REF_MODE[opts[1]], pc.REF_INTERP[opts[2]])
    assert h
    return r, h


def ref_process(r, h, fmt, ch, x, n, cap):
    y = np.full(pc.n_bytes(fmt, cap, ch), 7, dtype=np.uint8)
    got = r.ref_ars_process_packed(h, x.ctypes.data if x is not None else None, n, y.ctypes.data, cap)
    return got, y


# ---- the oracle against the reference build ---------------------------------------------------------------------------

@need_ref
@pytest.mark.parametrize("fmt", pc.NAMES)
def test_oracle_matches_reference(fmt):
    """every option set of the emulated kernel tests x FULL / interpolated / small-method / copy plans: buffers of 300,
    100 and 1 frames and a drain, byte for byte"""
    for opts in pc.OPTS:
        for (a, b, ch, q) in rates_for(opts):
            o = pc.OraclePacked(a, b, ch, q, fmt, opts)
            r, h = ref_stream(a, b, ch, q, fmt, opts)
            rng = np.random.default_rng(a + ch + q)
            try:
                for n in [300, 100, 1, None]:
                    x = None if n is None else pc.packed_signal(rng, n, ch, fmt)
                    n = 64 if n is None else n
                    cap = int(n * b / a) + 64
                    n1, y1 = o.process(x, n, cap)
                    n2, y2 = ref_process(r, h, fmt, ch, x, n, cap)
                    assert n1 == n2 and y1.tobytes() == y2.tobytes(), (opts, a, b, n)
            finally:
                o.free()
                r.ref_ars_free_packed(h)


@need_ref
@pytest.mark.parametrize("fmt", [f for f in pc.NAMES if not pc.FORMATS[f][6]])
def test_full_scale_saturates_like_reference(fmt):
    """a full-scale square wave: the filter's overshoot takes the S32 result to the top, where the quantizer's bias
    saturates (addssl), and the unsigned formats' sign flip sits on every sample"""
    a, b, ch, q = 48000, 44100, 2, 4
    _, w, step, depth, signed, big, _ = pc.FORMATS[fmt]
    top, bottom = ((1 << (depth - 1)) - 1, 1 << (depth - 1)) if signed else ((1 << depth) - 1, 0)
    codes = np.tile(np.repeat(np.array([top, bottom], dtype=np.uint64), 40), 8)
    x = np.zeros(len(codes) * 2 * w, dtype=np.uint8)
    order = range(step - 1, -1, -1) if big else range(step)
    for c in range(2):
        for j, bi in enumerate(order):
            x[(np.arange(len(codes)) * 2 + c) * step + bi] = ((codes >> np.uint64(8 * j)) & np.uint64(0xFF)).astype(np.uint8)
    o = pc.OraclePacked(a, b, ch, q, fmt)
    r, h = ref_stream(a, b, ch, q, fmt, pc.OPTS[0])
    try:
        n = len(codes)
        n1, y1 = o.process(x, n, n)
        n2, y2 = ref_process(r, h, fmt, ch, x, n, n)
        assert n1 == n2 > 0 and y1.tobytes() == y2.tobytes()
    finally:
        o.free()
        r.ref_ars_free_packed(h)


@need_ref
@pytest.mark.parametrize("fmt", ["U8", "S24LE", "S20_32BE", "F32BE"])
def test_stream_reset_and_update_match_reference(fmt):
    """many buffers, a reset, a drain, and rate updates across a FULL <-> interpolated switch (48k -> 44.1k has a phase
    table, 44.1k -> 48001 does not) with the history carried over"""
    ch, q = 2, 4
    o = pc.OraclePacked(48000, 44100, ch, q, fmt)
    r, h = ref_stream(48000, 44100, ch, q, fmt, pc.OPTS[0])
    ro, rr = o.resampler(), r.ref_ars_packed_resampler(h)
    rng = np.random.default_rng(5)
    try:
        for step, (a, b) in enumerate([(48000, 44100), (44100, 48001), (48000, 44100), (48000, 32000)]):
            if step:
                assert pc.oracle().oracle_ars_update(ro, a, b) == 0
                assert r.ref_ars_update(rr, a, b, q, 4, 2, 2) == 0
            if step == 2:
                pc.oracle().oracle_ars_reset(ro)
                r.ref_ars_reset(rr)
            for n in [int(v) for v in rng.choice([1, 33, 160, 481], 3)] + [None]:
                x = None if n is None else pc.packed_signal(rng, n, ch, fmt)
                n = 50 if n is None else n
                cap = int(n * b / a) + 64
                n1, y1 = o.process(x, n, cap)
                n2, y2 = ref_process(r, h, fmt, ch, x, n, cap)
                assert n1 == n2 and y1.tobytes() == y2.tobytes(), (step, a, b, n)
    finally:
        o.free()
        r.ref_ars_free_packed(h)


def test_s16be_is_not_a_byte_swapped_s16le():
    """S16BE runs through the S32 arithmetic and quantizer, S16LE through the S16 one: on the same samples the outputs
    differ beyond byte order, so a byte swap around the S16 kernels would not be the reference"""
    from oracle import bindings as ob
    a, b, ch, q = 48000, 44100, 2, 4
    rng = np.random.default_rng(3)
    x16 = ob.audio_test_signal(rng, 480, ch, "S16")
    xbe = np.frombuffer(x16.astype(">i2").tobytes(), dtype=np.uint8).copy()
    o = pc.OraclePacked(a, b, ch, q, "S16BE")
    ho = pc.oracle().oracle_ars_new_fmt(a, b, ch, q, 1)
    try:
        n1, ybe = o.process(xbe, 480, 480)
        y16 = np.zeros((480, ch), dtype=np.int16)
        n2 = pc.oracle().oracle_ars_process_any(ho, x16.ctypes.data, 480, y16.ctypes.data, 480)
        assert n1 == n2 > 0
        swapped = np.frombuffer(ybe[:n1 * ch * 2].tobytes(), dtype=">i2").reshape(n1, ch)
        assert (swapped != y16[:n1]).any()
    finally:
        o.free()
        pc.oracle().oracle_ars_free(ho)


# ---- the golden fixture -------------------------------------------------------------------------------------------------

def golden():
    cs = json.load(open(os.path.join(ROOT, "tests", "golden", "audio_packed_cases.json")))
    return cs, np.load(os.path.join(ROOT, "tests", "golden", "audio_packed.npz"))


def test_oracle_matches_golden():
    cs, z = golden()
    for i, c in enumerate(cs["cases"]):
        (a, b), ch, fmt = c["rates"], c["channels"], c["fmt"]
        o = pc.OraclePacked(a, b, ch, c["quality"], fmt, tuple(c["opts"]))
        try:
            for j, n in enumerate(cs["calls"]):
                x = z["c%d_in%d" % (i, j)] if n is not None else None
                n = pc.oracle().oracle_ars_max_latency(o.resampler()) if n is None else n
                got, y = o.process(x, n, int(n * b / a) + 64)
                want = z["c%d_out%d" % (i, j)]
                assert y[:len(want)].tobytes() == want.tobytes() and len(want) == pc.n_bytes(fmt, got, ch), (c, j)
        finally:
            o.free()


# ---- the product: host plan, launches, emulated kernels -----------------------------------------------------------------

@pytest.fixture(scope="module")
def emu():
    import build_emu
    from gstreamer_b200 import _lib
    lib = C.CDLL(build_emu.build())
    for name, (res, args) in _lib._SIGS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return lib


def plan(lib, cfg):
    from gstreamer_b200 import _lib
    h = C.c_void_p()
    assert lib.b200_ars_create(C.byref(cfg), -1, C.byref(h)) == 0
    i = _lib.ArsPlanInfoC()
    try:
        assert lib.b200_ars_get_plan_info(h, C.byref(i)) == 0
        return [i.n_taps, i.n_phases, i.in_step, i.out_step, i.filter_mode, i.oversample]
    finally:
        lib.b200_ars_destroy(h)


@pytest.mark.parametrize("rates", [(48000, 44100, 4), (44100, 48001, 4), (96000, 8000, 7), (44100, 48000, 10)])
def test_host_plan_is_the_intermediate_plan(emu, rates):
    """the plan (taps, phases, FULL or interpolated) of a packed format is that of its unpack format: the FULL-mode
    threshold counts the 4- or 8-byte intermediate samples, not the packed width"""
    a, b, q = rates
    s32 = plan(emu, pc.config(None, a, b, 2, q, 12))
    f64 = plan(emu, pc.config(None, a, b, 2, q, 30))
    for fmt in pc.NAMES:
        assert plan(emu, pc.config(None, a, b, 2, q, fmt)) == (f64 if pc.FORMATS[fmt][6] else s32), fmt
    for bad in (0 + 1, 36, 40, -3):
        h = C.c_void_p()
        assert emu.b200_ars_create(C.byref(pc.config(None, a, b, 2, q, bad)), -1, C.byref(h)) == -2


def test_launches_match_fixture():
    import make_ars_packed_routes as mp
    want = json.load(open(mp.FIXTURE))
    got = json.loads(json.dumps(mp.record(), sort_keys=True))
    assert got == want
    names = {x.split(" grid=")[0] for row in got.values() if len(row) > 1 for i in (2, 4) for call in row[i] for x in call[2]}
    assert names == {"ars_direct_kernel_packed<2, true>", "ars_direct_kernel_packed<2, false>",
                     "ars_direct_kernel_packed<3, true>", "ars_direct_kernel_packed<3, false>",
                     "ars_small_kernel_packed<2>", "ars_small_kernel_packed<3>",
                     "ars_history_kernel_packed<int>", "ars_history_kernel_packed<double>"}


def emu_stream(emu, a, b, ch, q, fmt, opts=pc.OPTS[0]):
    h = C.c_void_p()
    assert emu.b200_ars_create(C.byref(pc.config(None, a, b, ch, q, fmt, opts)), 0, C.byref(h)) == 0
    return h


def emu_process(emu, h, fmt, ch, x, n, cap, host=False):
    y = np.full(pc.n_bytes(fmt, cap, ch), 7, dtype=np.uint8)
    got = C.c_size_t()
    xp = x.ctypes.data if x is not None else None
    if host:
        assert emu.b200_ars_process_host(h, xp, n, y.ctypes.data, cap, C.byref(got)) == 0
    else:
        assert emu.b200_ars_process(h, xp, n, y.ctypes.data, cap, C.byref(got), None) == 0
    return got.value, y


EMU_OPTS = [pc.OPTS[0], pc.OPTS[1], pc.OPTS[3], pc.OPTS[6], pc.OPTS[7], pc.OPTS[9], pc.OPTS[10], pc.OPTS[11]]


@pytest.mark.parametrize("fmt", pc.NAMES)
def test_emulated_kernels_match_oracle(emu, fmt):
    """ars_direct_kernel_packed / ars_small_kernel_packed / ars_history_kernel_packed byte for byte against the oracle:
    FULL, interpolated, small-method and copy plans, several buffers, a one-frame call and a drain; nothing is written
    past the frames produced"""
    for opts in EMU_OPTS:
        for (a, b, ch, q) in rates_for(opts):
            o = pc.OraclePacked(a, b, ch, q, fmt, opts)
            h = emu_stream(emu, a, b, ch, q, fmt, opts)
            rng = np.random.default_rng(a + ch)
            try:
                for n in [300, 100, 1, None]:
                    x = None if n is None else pc.packed_signal(rng, n, ch, fmt)
                    n = emu.b200_ars_get_max_latency(h) if n is None else n
                    cap = int(n * b / a) + 64
                    n1, y1 = o.process(x, n, cap)
                    n2, y2 = emu_process(emu, h, fmt, ch, x, n, cap)
                    assert n1 == n2 and y1.tobytes() == y2.tobytes(), (opts, a, b, ch, n)
            finally:
                emu.b200_ars_destroy(h)
                o.free()


@pytest.mark.parametrize("fmt", ["U8", "S16BE", "S24LE", "S24_32BE", "F32BE", "S20_32LE"])
def test_emulated_reset_and_update(emu, fmt):
    """b200_ars_update across a FULL <-> interpolated switch (history moved in the intermediate format) and
    b200_ars_reset, against the oracle"""
    ch, q = 3, 4
    o = pc.OraclePacked(48000, 44100, ch, q, fmt)
    h = emu_stream(emu, 48000, 44100, ch, q, fmt)
    rng = np.random.default_rng(11)
    try:
        for step, (a, b) in enumerate([(48000, 44100), (44100, 48001), (48000, 44100), (48000, 32000)]):
            if step:
                assert pc.oracle().oracle_ars_update(o.resampler(), a, b) == 0
                assert emu.b200_ars_update(h, a, b) == 0
            if step == 2:
                pc.oracle().oracle_ars_reset(o.resampler())
                assert emu.b200_ars_reset(h) == 0
            for n in [int(v) for v in rng.choice([1, 7, 160, 481], 3)]:
                x = pc.packed_signal(rng, n, ch, fmt)
                cap = int(n * b / a) + 64
                n1, y1 = o.process(x, n, cap)
                n2, y2 = emu_process(emu, h, fmt, ch, x, n, cap)
                assert n1 == n2 and y1.tobytes() == y2.tobytes(), (step, a, b, n)
    finally:
        emu.b200_ars_destroy(h)
        o.free()


@pytest.mark.parametrize("fmt", ["U8", "S24LE", "F64BE", "S20_32BE"])
def test_emulated_host_path_equals_device_path(emu, fmt):
    """b200_ars_process_host stages the caller's packed bytes (packed width per sample) and gives the device path's bytes"""
    a, b, ch, q = 44100, 48000, 2, 4
    hh, hd = emu_stream(emu, a, b, ch, q, fmt), emu_stream(emu, a, b, ch, q, fmt)
    rng = np.random.default_rng(2)
    try:
        for n in (2000, 480, 1300):
            x = pc.packed_signal(rng, n, ch, fmt)
            cap = emu.b200_ars_get_out_frames(hd, n)
            n1, y1 = emu_process(emu, hh, fmt, ch, x, n, cap, host=True)
            n2, y2 = emu_process(emu, hd, fmt, ch, x, n, cap)
            assert n1 == n2 > 0 and y1.tobytes() == y2.tobytes()
    finally:
        emu.b200_ars_destroy(hh)
        emu.b200_ars_destroy(hd)
