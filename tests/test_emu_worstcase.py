"""Worst-case content (tests/worstcase.py) through the product's kernels without a GPU (the emulated library,
tests/cudaemu): every batch row the emulator can run - every kernel of GRID_KERNELS - on batches of distinct worst-case
frames, with the launch sequence each row logs, and the resampler's routes under the knobs that select them on
full-scale streams, each case with the kernel its knobs select.  tests/test_worstcase_gpu.py runs the same content on the H100."""
import ctypes as C

import numpy as np
import pytest

import vcs_batch_cases as vb
import worstcase as wc
from oracle import bindings as ob
from test_emu_batch import EMU_ROWS, emu, launches  # noqa: F401  (emu is a fixture)
from test_vcs_routes import GRID_KERNELS

pytestmark = pytest.mark.timeout(600)           # emulated barriers: a logic error must fail, not hang the CPU suite


def test_rows_cover_the_grid():
    assert vb.kernels(EMU_ROWS) == GRID_KERNELS


@pytest.mark.parametrize("row", EMU_ROWS + wc.KNOB_ROWS, ids=lambda r: r.id)
def test_row_worst_case(emu, row, monkeypatch):
    """the row's launch sequence, then batches of 2 and 3 distinct worst-case frames on one handle"""
    mem = vb.HostMem()
    h = wc.WorstHandle(emu, row, monkeypatch)
    try:
        assert launches(emu, h, mem) == row.launches
        vb.check_batches(h, mem, (2, 3), seed=100)
    finally:
        h.close()


# (format, (in, out, channels, quality), knobs, the resampling kernel it must launch): the persistent pipelines and the
# tile shapes (128 channels), the small-channel kernels, the interpolated filter mode, the generic / direct kernels
ARS_CASES = [
    ("F32", (48000, 44100, 128, 4), None, "ars_pipe_kernel"),
    ("F32", (48000, 44100, 128, 4), "B200_ARS_PIPE_V1=1", "ars_pipe_kernel_v1"),
    ("F32", (48000, 44100, 128, 4), "B200_ARS_NOPIPE=1 B200_ARS_CPT=4", "ars_tile_kernel<128, 4>"),
    ("F32", (48000, 44100, 128, 4), "B200_ARS_NOPIPE=1 B200_ARS_CPT=1", "ars_tile_kernel<128, 1>"),
    ("F32", (48000, 44100, 128, 4), "B200_ARS_NOPIPE=1 B200_ARS_CB=32 B200_ARS_NO=16", "ars_tile_kernel<32, 1>"),
    ("F32", (48000, 44100, 128, 4), "B200_ARS_GENERIC=1", "ars_full_kernel"),
    ("S16", (48000, 44100, 128, 4), None, "ars_pipe_kernel_s16"),
    ("S16", (48000, 44100, 128, 4), "B200_ARS_NOPIPE=1", "ars_tile_kernel_s16<128>"),
    ("S16", (48000, 44100, 2, 4), "B200_ARS_GENERIC=1", "ars_direct_kernel<1, false>"),
    ("F32", (48000, 44100, 2, 4), None, "ars_tile_kernel<32, 1>"),
    ("F32", (48000, 44100, 2, 4), "B200_ARS_NO=64", "ars_tile_kernel<32, 1>"),
    ("F32", (44100, 48001, 2, 4), None, "ars_interp_kernel<false>"),
] + [(f, cfg, None, k) for f, k in (("S16", "ars_direct_kernel<1, false>"), ("S32", "ars_direct_kernel<2, false>"),
                                    ("F64", "ars_direct_kernel<3, false>"))
     for cfg in ((48000, 44100, 2, 4), (44100, 48001, 2, 4))]


def _ars_id(c):
    f, (a, b, ch, q), k, _ = c
    return "%s-%d-%d-%dch-q%d%s" % (f, a, b, ch, q, "" if k is None else "-" + k.replace(" ", "-"))


def ars_launches(emu, fmt, cfg):
    """the kernels (template arguments kept) two 1000-frame calls of a fresh handle launch (record-only: logged, not run)"""
    from gstreamer_b200 import _lib
    a, b, ch, q = cfg
    _, gfmt, dt, _ = ob.AUDIO_FORMATS[fmt]
    c = _lib.ArsConfigC()
    c.in_rate, c.out_rate, c.channels, c.quality, c.format = a, b, ch, q, gfmt
    h = C.c_void_p()
    assert emu.b200_ars_create(C.byref(c), 0, C.byref(h)) == 0
    x = np.zeros((1000, ch), dtype=dt)
    cap = int(1000 * b / a) + 64
    y = np.zeros((cap, ch), dtype=dt)
    ng = C.c_size_t()
    emu.b200emu_clear_launch_log()
    emu.b200emu_set_record_only(1)
    try:
        for _ in range(2):
            assert emu.b200_ars_process(h, x.ctypes.data, 1000, y.ctypes.data, cap, C.byref(ng), None) == 0
        return {x for x in emu.b200emu_launch_log().decode().split("\n") if x}
    finally:
        emu.b200emu_set_record_only(0)
        emu.b200emu_clear_launch_log()
        emu.b200_ars_destroy(h)


@pytest.mark.parametrize("case", ARS_CASES, ids=_ars_id)
def test_audio_worst_case(emu, monkeypatch, case):
    from gstreamer_b200 import _lib
    fmt, cfg, knobs, kernel = case
    for kv in (knobs or "").split():
        monkeypatch.setenv(*kv.split("="))
    a, b, ch, q = cfg
    _, gfmt, dt, _ = ob.AUDIO_FORMATS[fmt]
    assert kernel in ars_launches(emu, fmt, cfg)
    for scale in sorted({wc.ars_scale(fmt, cfg), 1.0}):
        c = _lib.ArsConfigC()
        c.in_rate, c.out_rate, c.channels, c.quality, c.format = a, b, ch, q, gfmt
        h = C.c_void_p()
        assert emu.b200_ars_create(C.byref(c), 0, C.byref(h)) == 0

        def transform(chunk, n, cap):
            got = np.full((cap, ch), 7, dtype=dt)
            ng = C.c_size_t()
            assert emu.b200_ars_process(h, chunk.ctypes.data if chunk is not None else None, n, got.ctypes.data, cap,
                                        C.byref(ng), None) == 0
            assert (got[ng.value:] == 7).all()
            return ng.value, got

        try:
            y, aims, full = wc.run_ars_case(transform, fmt, cfg, scale, seed=ch + q, n_total=3000)
        finally:
            emu.b200_ars_destroy(h)
        if fmt in ("F32", "F64") or (scale < 1.0 and full):
            assert wc.check_saturation(y, aims, fmt) > 0
