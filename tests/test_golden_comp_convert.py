"""Compositor convert pads against the REFERENCE build's bytes (tests/golden/comp_convert.npz, make_comp_convert.py: the
option-less GstVideoConverter of a GstVideoAggregatorConvertPad to the output's format and colorimetry, then the
reference blend), through b200_comp_blend_convert on the emulated library (tests/cudaemu).  Some outputs carry BT709 /
full range on a small frame: their converted pads must follow the output's colorimetry, not their own size's default."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tests", "cudaemu"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import comp_convert_cases as cc  # noqa: E402

pytestmark = pytest.mark.timeout(900)
CASES = json.load(open(os.path.join(G, "comp_convert_cases.json")))


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


class HostMem:
    def __init__(self):
        self.keep = []

    def upload(self, a):
        a = np.ascontiguousarray(a)
        self.keep.append(a)
        return a.ctypes.data, a

    def download(self, a):
        return a.copy()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["key"])
def test_reference_bytes(emu, case):
    gold = np.load(os.path.join(G, "comp_convert.npz"))[case["key"]]
    mem = HostMem()
    s = cc.Setup(emu, mem, case)
    try:
        assert s.call() == 0
        got = cc.unpack(case["out"], mem.download(s.dst), s.di)
    finally:
        s.close()
    cc.check_bytes(got, gold, case["key"])
