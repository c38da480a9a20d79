"""b200_comp_blend_convert on the device: the random-layout grid of tests/test_comp_convert.py, the mosaic workloads at
full size and pitched GstCudaMemory-style layouts, byte for byte against oracle_vcs_convert + oracle_compositor[_yuv],
with the route each pad takes (comp_convert_cases.Setup.routes) asserted per configuration."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import comp_convert_cases as cc  # noqa: E402

pytestmark = pytest.mark.gpu


class TorchMem:
    def __init__(self):
        import torch
        self.torch = torch
        self.keep = []

    def upload(self, a):
        t = self.torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.keep.append(t)
        return t.data_ptr(), t

    def download(self, t):
        self.torch.cuda.synchronize()
        return t.cpu().numpy()


@pytest.fixture(scope="module")
def lib(cuda_device):
    from gstreamer_b200._lib import lib
    return lib


def run(lib, case):
    mem = TorchMem()
    s = cc.Setup(lib, mem, case)
    try:
        routes = s.routes()
        assert s.call() == 0
        got = cc.unpack(case["out"], mem.download(s.dst), s.di)
        return got, s.expected(), routes
    finally:
        s.close()


@pytest.mark.parametrize("out_name", ["I420", "YV12", "NV12", "NV21", "BGRA", "RGBA", "ARGB", "ABGR"])
def test_random_layouts(lib, out_name):
    rng = np.random.default_rng(100 + cc.FMT[out_name])
    seen = set()
    for trial in range(12):
        case = cc.random_case(rng, out_name, trial, max_size=(300, 200), max_pads=8 if trial < 10 else 40,
                              min_pads=0 if trial < 10 else 36, pad_max=None if trial < 10 else (60, 40))
        got, want, routes = run(lib, case)
        cc.check_bytes(got, want, f"{out_name} trial {trial} routes {routes}")
        seen.update(routes)
    if out_name in cc.YUV420:
        assert {"fused", "blend", "two-pass"} <= seen, seen
    else:
        assert "fused" not in seen and {"blend", "two-pass"} <= seen, seen


@pytest.mark.parametrize("name", ["M1", "M2", "M3"])
def test_mosaic_workloads(lib, name):
    """M1: 16 x 1080p NV12 at 960x540 in a 4 x 4 grid -> 3840x2160 NV12; M2: 9 at 640x360 -> 1080p NV12 plus one 1080p pad
    on top at alpha 0.5; M3: 4 at 960x540 -> 1080p BGRA"""
    if name == "M1":
        case = cc.mosaic_case("NV12", tile=(960, 540), src=(1920, 1080), grid=(4, 4))
    elif name == "M2":
        case = cc.mosaic_case("NV12", tile=(640, 360), src=(1920, 1080), grid=(3, 3))
        case["pads"].append(cc.pad("NV12", 1920, 1080, 640, 360, 320, 180, alpha=0.5, seed=99))
    else:
        case = cc.mosaic_case("BGRA", tile=(960, 540), src=(1920, 1080), grid=(2, 2), in_fmt="NV12")
    got, want, routes = run(lib, case)
    cc.check_bytes(got, want, name)
    assert set(routes) == ({"two-pass"} if name == "M3" else {"fused"}), routes


@pytest.mark.parametrize("out_name", ["NV12", "I420"])
def test_pitched_layouts(lib, out_name):
    """GstCudaMemory-style layouts (one pitch for all planes, pitch-aligned plane offsets) for the destination and every pad"""
    case = cc.mosaic_case(out_name, tile=(100, 60), src=(150, 90), grid=(3, 2))
    case["pads"][1]["alpha"] = 0.5
    case["pads"].append(cc.pad(out_name, 64, 40, 64, 40, 21, 9, alpha=0.5, seed=7))
    case["dst_odd"] = "pitch"
    for p in case["pads"]:
        p["odd"] = "pitch"
    got, want, routes = run(lib, case)
    cc.check_bytes(got, want, "pitched")
    assert routes == ["fused"] * 6 + ["blend"], routes



GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("case", json.load(open(os.path.join(GOLDEN, "comp_convert_cases.json"))), ids=lambda c: c["key"])
def test_reference_bytes(lib, case):
    """the reference build's bytes (tests/golden/make_comp_convert.py), outputs with a colorimetry of their own included"""
    gold = np.load(os.path.join(GOLDEN, "comp_convert.npz"))[case["key"]]
    got, _, _ = run(lib, case)
    cc.check_bytes(got, gold, case["key"])
