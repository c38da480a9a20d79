"""The converter's batch dimension without a GPU: every row of tests/vcs_batch_cases.py that the emulated library
(tests/cudaemu) can run - all but vcs_l2tc_kernel - on batches of distinct frames, against the oracle.  Each row first
checks the launch sequence its handle logs, so that together the rows run every kernel a convert can launch on more than
one frame.  tests/test_vcs_batch_gpu.py runs the same rows on the H100."""
import ctypes as C
import os
import sys

import pytest

import vcs_batch_cases as vb
from test_vcs_routes import GRID_KERNELS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "cudaemu"))

pytestmark = pytest.mark.timeout(600)           # emulated barriers: a logic error must fail, not hang the CPU suite

EMU_ROWS = [r for r in vb.ROWS if not r.device_only]


@pytest.fixture(scope="module")
def emu():
    import build_emu
    from gstreamer_b200 import _lib
    lib = C.CDLL(build_emu.build())
    for name, (res, args) in _lib._SIGS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    lib.b200emu_launch_log.restype = C.c_char_p
    lib.b200emu_set_record_only.argtypes = [C.c_int]
    return lib


def launches(emu, h, mem):
    """the kernels one convert of a two-frame batch launches (record-only: logged, not run)"""
    ins, outs = [mem.buffer(h.in_size) for _ in range(2)], [mem.buffer(h.out_size) for _ in range(2)]
    emu.b200emu_clear_launch_log()
    emu.b200emu_set_record_only(1)
    try:
        assert h.convert([mem.ptr(b) for b in ins], [mem.ptr(b) for b in outs]) == 0
        log = emu.b200emu_launch_log().decode()
    finally:
        emu.b200emu_set_record_only(0)
        emu.b200emu_clear_launch_log()
    return tuple(x for x in log.split("\n") if x)


def test_rows_launch_every_kernel():
    """the emulated rows launch every kernel the route grid reaches (tests/test_vcs_routes.py), the device rows
    vcs_l2tc_kernel as well: a kernel added to the converter needs a batch row"""
    assert vb.kernels(EMU_ROWS) == GRID_KERNELS
    assert vb.kernels(vb.ROWS) == GRID_KERNELS | {"vcs_l2tc_kernel"}
    assert len({r.id for r in vb.ROWS}) == len(vb.ROWS)


@pytest.mark.parametrize("row", EMU_ROWS, ids=lambda r: r.id)
def test_batch_row(emu, row, monkeypatch):
    """the row's launch sequence; then, on one handle: batches of 2, 5 and 3 distinct frames (the scratch image grows,
    then its slices are reused), frames at shuffled offsets of one allocation, one input twice, and a refused 65-frame
    batch"""
    mem = vb.HostMem()
    h = vb.Handle(emu, row, monkeypatch)
    try:
        got = launches(emu, h, mem)
        print(f"{row.id}: {' -> '.join(got)}")
        assert got == row.launches, got
        vb.check_batches(h, mem, (2, 5, 3), seed=11)
        vb.check_unordered(h, mem, 5, seed=21)
        vb.check_aliased_input(h, mem, seed=31)
        vb.check_too_many(h, mem, seed=41)
    finally:
        h.close()


def test_batch_of_64(emu, monkeypatch):
    """a full batch (B200_VCS_MAX_BATCH distinct frames) on the smallest rows: a chain with its scratch image and
    vcs_down420_kernel, and the plane copy"""
    mem = vb.HostMem()
    for rid in ("nv12-i420-odd-height", "i420-i420-copy"):
        h = vb.Handle(emu, next(r for r in EMU_ROWS if r.id == rid), monkeypatch)
        try:
            vb.check_batches(h, mem, (vb.MAX_BATCH,), seed=51)
        finally:
            h.close()
