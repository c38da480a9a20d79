"""cudaaudioresample's packed sample formats on the device, byte for byte against the oracle: one format of each storage
class (tests/ars_packed_cases.py CLASSES) with 1, 2, 6 and 256 channels, input and output at odd byte offsets, streams
with a drain, a reset and a rate update across a FULL <-> interpolated switch, and the system-memory path."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ars_packed_cases as pc  # noqa: E402

pytestmark = pytest.mark.gpu


def device_process(lib, h, fmt, ch, x, n, cap, off_in, off_out):
    """one b200_ars_process call with the input and output `off_in` / `off_out` bytes into their device buffers"""
    import torch
    nb = pc.n_bytes(fmt, n, ch)
    din = torch.zeros(nb + 16, dtype=torch.uint8, device="cuda")
    if x is not None:
        din[off_in:off_in + nb] = torch.from_numpy(x).cuda()
    ob = pc.n_bytes(fmt, cap, ch)
    dout = torch.full((ob + 16,), 7, dtype=torch.uint8, device="cuda")
    got = C.c_size_t()
    st = lib.b200_ars_process(h, din.data_ptr() + off_in if x is not None else None, n, dout.data_ptr() + off_out, cap,
                              C.byref(got), None)
    assert st == 0
    torch.cuda.synchronize()
    y = dout.cpu().numpy()
    assert (y[:off_out] == 7).all() and (y[off_out + ob:] == 7).all()
    return got.value, y[off_out:off_out + ob]


def create(lib, a, b, ch, q, fmt, opts=pc.OPTS[0]):
    h = C.c_void_p()
    assert lib.b200_ars_create(C.byref(pc.config(None, a, b, ch, q, fmt, opts)), 0, C.byref(h)) == 0
    return h


@pytest.mark.parametrize("ch", [1, 2, 6, 256])
@pytest.mark.parametrize("fmt", pc.CLASSES)
def test_packed_stream_matches_oracle(fmt, ch):
    from gstreamer_b200._lib import lib
    for opts, (a, b, q) in [(pc.OPTS[0], (48000, 44100, 4)), (pc.OPTS[7], (44100, 48001, 4)), (pc.OPTS[11], (3, 2, 5)),
                            (pc.OPTS[0], (44100, 44100, 4))]:
        o = pc.OraclePacked(a, b, ch, q, fmt, opts)
        h = create(lib, a, b, ch, q, fmt, opts)
        rng = np.random.default_rng(ch + a)
        try:
            for k, n in enumerate([2000, 333, 1, None]):
                x = None if n is None else pc.packed_signal(rng, n, ch, fmt)
                n = lib.b200_ars_get_max_latency(h) if n is None else n
                cap = int(n * b / a) + 64
                n1, y1 = o.process(x, n, cap)
                n2, y2 = device_process(lib, h, fmt, ch, x, n, cap, (1, 3, 0, 5)[k], (3, 1, 7, 0)[k])
                assert n1 == n2 and y1.tobytes() == y2.tobytes(), (opts, a, b, n)
        finally:
            lib.b200_ars_destroy(h)
            o.free()


@pytest.mark.parametrize("fmt", ["U8", "S24LE", "S20_32BE", "F32BE"])
def test_packed_update_and_reset_match_oracle(fmt):
    from gstreamer_b200._lib import lib
    ch, q = 6, 4
    o = pc.OraclePacked(48000, 44100, ch, q, fmt)
    h = create(lib, 48000, 44100, ch, q, fmt)
    rng = np.random.default_rng(9)
    try:
        for step, (a, b) in enumerate([(48000, 44100), (44100, 48001), (48000, 44100), (48000, 32000)]):
            if step:
                assert pc.oracle().oracle_ars_update(o.resampler(), a, b) == 0
                assert lib.b200_ars_update(h, a, b) == 0
            if step == 2:
                pc.oracle().oracle_ars_reset(o.resampler())
                assert lib.b200_ars_reset(h) == 0
            for n in [int(v) for v in rng.choice([1, 7, 160, 4801], 3)]:
                x = pc.packed_signal(rng, n, ch, fmt)
                cap = int(n * b / a) + 64
                n1, y1 = o.process(x, n, cap)
                n2, y2 = device_process(lib, h, fmt, ch, x, n, cap, 3, 1)
                assert n1 == n2 and y1.tobytes() == y2.tobytes(), (step, a, b, n)
    finally:
        lib.b200_ars_destroy(h)
        o.free()


@pytest.mark.parametrize("fmt", ["U8", "S24LE", "F64BE", "S20_32LE"])
def test_packed_host_path_matches_oracle(fmt):
    """b200_ars_process_host: pageable host buffers of packed samples, the staging ring sized by the packed width"""
    from gstreamer_b200._lib import lib
    a, b, ch, q = 44100, 48000, 256, 4
    o = pc.OraclePacked(a, b, ch, q, fmt)
    h = create(lib, a, b, ch, q, fmt)
    rng = np.random.default_rng(4)
    try:
        for n in (4410, 480, 1300):
            x = pc.packed_signal(rng, n, ch, fmt)
            cap = lib.b200_ars_get_out_frames(h, n)
            n1, y1 = o.process(x, n, cap)
            y2 = np.full(len(y1), 7, dtype=np.uint8)
            got = C.c_size_t()
            assert lib.b200_ars_process_host(h, x.ctypes.data, n, y2.ctypes.data, cap, C.byref(got)) == 0
            assert got.value == n1 and y1.tobytes() == y2.tobytes()
    finally:
        lib.b200_ars_destroy(h)
        o.free()
