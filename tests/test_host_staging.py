"""The system-memory ("host") entry points on the emulated library (tests/cudaemu), without a GPU: what each call issues
(the level-3 log of tests/golden/host_staging.json, tests/golden/make_host_staging.py), the bytes each gives against its
device-memory call on the same frames, and a staging setup that fails part way: the call fails, leaves nothing behind,
and the next call sets the ring up again from scratch."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import make_host_staging as mh  # noqa: E402

pytestmark = pytest.mark.timeout(900)


@pytest.fixture(scope="module")
def emu():
    return mh.Emu()


def test_staging_matches_fixture(emu):
    got = json.loads(json.dumps(mh.record()))
    want = json.load(open(mh.FIXTURE))
    assert got.keys() == want.keys()
    for k in want:
        assert got[k]["calls"] == want[k]["calls"], k
        assert got[k]["log"] == want[k]["log"], k


# ---- one call on the host path and on device memory, kernels running (level 0) --------------------------------------

def vcs_pair(e, mem, h, ib, ob, n):
    rc, ins, outs = e.convert_host(h, mem, n, ib, ob)
    assert rc == 0
    dev = [mem.buf(ob) for _ in range(n)]
    for i0 in range(0, n, 64):
        m = min(64, n - i0)
        assert e.lib.b200_vcs_convert_batch(h, m, mem.ptrs(ins[i0:i0 + m]), mem.ptrs(dev[i0:i0 + m]), None) == 0
    return outs, dev


def comp_rgb_pair(e, mem, h, W, H, specs):
    pads = e.rgb_pads(mem, specs)
    a, b = mem.buf(W * 4 * H), mem.buf(W * 4 * H)
    assert e.lib.b200_comp_blend_host(h, a.ctypes.data, W * 4, 0, pads, len(specs)) == 0
    assert e.lib.b200_comp_blend(h, b.ctypes.data, W * 4, 0, pads, len(specs), None) == 0
    return [a], [b]


def comp_yuv_pair(e, mem, h, fmt, W, H, specs):
    pads = e.yuv_pads(mem, fmt, specs)
    di = e.info(fmt, W, H, 8)
    a = mem.buf(e.size(di))
    b = a.copy()
    mem.keep.append(b)
    assert e.lib.b200_comp_blend_yuv_host(h, a.ctypes.data, C.byref(di), 1, pads, len(specs)) == 0
    assert e.lib.b200_comp_blend_yuv(h, b.ctypes.data, C.byref(di), 1, pads, len(specs), None) == 0
    return [a], [b]


def ars_pair(e, mem, hh, hd, n, bpf):
    src = mem.buf(n * bpf)
    want = e.lib.b200_ars_get_out_frames(hh, n)
    a, b = mem.buf(want * bpf), mem.buf(want * bpf)
    ga, gb = C.c_size_t(0), C.c_size_t(0)
    assert e.lib.b200_ars_process_host(hh, src.ctypes.data, n, a.ctypes.data, want, C.byref(ga)) == 0
    assert e.lib.b200_ars_process(hd, src.ctypes.data, n, b.ctypes.data, want, C.byref(gb), None) == 0
    assert ga.value == gb.value
    return [a[:ga.value * bpf]], [b[:gb.value * bpf]]


def same(pair):
    host, dev = pair
    assert len(host) == len(dev)
    for a, b in zip(host, dev):
        np.testing.assert_array_equal(a, b)


SMALL_VCS = ((mh.NV12, 32, 16), (mh.BGRA, 16, 8))


@pytest.mark.parametrize("n", [3, 33])
def test_vcs_host_equals_device(emu, n):
    mem = mh.Host(10)
    h, ib, ob = emu.vcs(SMALL_VCS)
    try:
        same(vcs_pair(emu, mem, h, ib, ob, n))
    finally:
        emu.lib.b200_vcs_destroy(h)


def test_comp_host_equals_device(emu):
    mem = mh.Host(11)
    h = emu.comp(mh.BGRA, 32, 24)
    try:
        for specs in mh.RGB_STEPS:
            same(comp_rgb_pair(emu, mem, h, 32, 24, specs))
    finally:
        emu.lib.b200_comp_destroy(h)


@pytest.mark.parametrize("fmt", mh.COMP_YUV)
def test_comp_yuv_host_equals_device(emu, fmt):
    mem = mh.Host(12)
    h = emu.comp(fmt, 32, 24)
    try:
        for specs in mh.RGB_STEPS[:5]:
            same(comp_yuv_pair(emu, mem, h, fmt, 32, 24, specs))
    finally:
        emu.lib.b200_comp_destroy(h)


@pytest.mark.parametrize("fmt", [mh.F32, mh.S16])
def test_ars_host_equals_device(emu, fmt):
    mem = mh.Host(13)
    bpf = 2 * (4 if fmt == mh.F32 else 2)
    hh, hd = emu.ars(fmt), emu.ars(fmt)
    try:
        for n in (2000, 480, 1300):
            same(ars_pair(emu, mem, hh, hd, n, bpf))
    finally:
        emu.lib.b200_ars_destroy(hh)
        emu.lib.b200_ars_destroy(hd)


# ---- a staging setup that fails at its k-th stream or event creation -------------------------------------------------

OWNERS = {"vcs": 4, "comp": 3, "ars": 3}                          # staging slots of each owner


def owner_call(e, mem, owner):
    """a fresh handle of the owner, its destroy, one host call against the device-memory call (host bytes, device
    bytes), and one host call alone (its status)"""
    if owner == "vcs":
        h, ib, ob = e.vcs(SMALL_VCS)
        return h, e.lib.b200_vcs_destroy, lambda: vcs_pair(e, mem, h, ib, ob, 2), \
            lambda: e.convert_host(h, mem, 2, ib, ob)[0]
    if owner == "comp":
        h = e.comp(mh.BGRA, 32, 24)
        return h, e.lib.b200_comp_destroy, lambda: comp_rgb_pair(e, mem, h, 32, 24, mh.RGB_STEPS[0]), \
            lambda: e.lib.b200_comp_blend_host(h, mem.buf(32 * 4 * 24).ctypes.data, 32 * 4, 0, e.rgb_pads(mem, mh.RGB_STEPS[0]), 2)
    h, hd = e.ars(mh.F32), e.ars(mh.F32)

    def destroy(x):
        e.lib.b200_ars_destroy(x)
        e.lib.b200_ars_destroy(hd)

    def call():                                                    # keeps the device-memory handle in step
        st = e.ars_submit(h, mem, 2000, 8)[0]
        if st == 0:
            out, got = mem.buf(2000 * 8), C.c_size_t(0)
            assert e.lib.b200_ars_process(hd, mem.buf(2000 * 8).ctypes.data, 2000, out.ctypes.data, 2000, C.byref(got), None) == 0
        return st
    return h, destroy, lambda: ars_pair(e, mem, h, hd, 2000, 8), call


def logged(e, fn):
    r = e.record(lambda: [fn()])
    return r["calls"][0], r["log"]


def count(log, prefix):
    return sum(1 for x in log if x.startswith(prefix))


@pytest.mark.parametrize("owner", sorted(OWNERS))
def test_failed_setup_starts_again(emu, owner):
    n_handles = 3 + 3 * OWNERS[owner]
    for k in range(1, n_handles + 1):
        mem = mh.Host(14)
        h, destroy, pair, call = owner_call(emu, mem, owner)
        try:
            emu.lib.b200emu_fail_create(k)
            st, log = logged(emu, call)
            emu.lib.b200emu_fail_create(0)
            assert st == -4, (k, st)                                # B200_ERR_CUDA
            made = count(log, "cudaStreamCreate s") + count(log, "cudaEventCreate e")
            assert made == k - 1 and count(log, "cudaStreamDestroy") + count(log, "cudaEventDestroy") == made, (k, log)
            st, log = logged(emu, call)
            assert st == 0, (k, st)
            assert count(log, "cudaStreamCreate s") == 3 and count(log, "cudaEventCreate e") == 3 * OWNERS[owner], (k, log)
            assert not any("failed" in x for x in log)
            same(pair())
        finally:
            emu.lib.b200emu_fail_create(0)
            destroy(h)
