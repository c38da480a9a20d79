"""The fused route's plane scalers without a GPU (tests/comp_fused_cases.py, the emulated library): every CompStore kernel
the library compiles is either launched by a row or unreachable for a stated rule; each row launches its form and, on
worst-case content of its own taps at clipped positions and alphas copy / 254 / 128 / 1, gives the bytes of
oracle_vcs_convert + oracle_compositor_yuv; comp_store's (p, v, a) domain through two byte-picking forms."""
import os

import numpy as np
import pytest

import comp_convert_cases as cc
import comp_domain as cd
import comp_fused_cases as cf
from test_comp_convert import EmuMem, emu  # noqa: F401  (emu is a fixture)

pytestmark = pytest.mark.timeout(900)

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gstreamer_b200", "libb200dsp.so")


def test_rows_and_unreachable_cover_the_library():
    forms = cf.library_forms(LIB)
    rows = {r.form for r in cf.ROWS}
    unreachable = {f for f in forms if cf.unreachable_reason(f)}
    assert rows <= forms, rows - forms
    assert not rows & unreachable, rows & unreachable
    assert rows | unreachable == forms, sorted(forms - rows - unreachable)


def run_row(lib, mem, case, form, log):
    if log is not None:
        assert form in cc.route_log(log, case), form
    got, want, routes = cc.run_case(lib, mem, case, None, log=log)
    cc.check_bytes(got, want, form)
    assert set(routes) == {"fused"}, routes


@pytest.mark.parametrize("row", cf.ROWS, ids=lambda r: f"{r.out}-{r.form}")
def test_row(emu, row):  # noqa: F811
    run_row(emu, EmuMem(), cf.row_case(row), row.form, emu)


def store_pairs(case):
    """the (p, v) pairs each alpha band of a store_case meets in the luma plane"""
    from oracle import bindings as ob
    p0 = case["pads"][0]
    W = case["W"]
    p = case["content"](p0)[: W * case["H"]].reshape(case["H"], W).astype(np.int64)
    out = []
    for pad in case["pads"][1:]:
        conv = ob.oracle_vcs_convert(ob.vcs_desc(pad["iw"], pad["ih"], pad["pw"], pad["ph"], 0, in_fmt=2, out_fmt=2),
                                     case["content"](pad))
        v = conv[: pad["pw"] * pad["ph"]].reshape(pad["ph"], pad["pw"]).astype(np.int64)
        band = p[pad["y"]: pad["y"] + pad["ph"]]
        out.append(np.unique(band * 256 + v).size)
    return out


EMU_STORE_ALPHAS = [cd.alpha_for(k, 255) for k in (1, 2, 127, 128, 129, 254, 255)] + [1.0]


@pytest.mark.parametrize("form", list(cf.STORE_FORMS))
def test_store_domain(emu, form):  # noqa: F811
    """every (p, v) at alphas 1, 2, 127, 128, 129, 254, 255 and copy (the GPU file runs every alpha)"""
    case = cf.store_case(form, EMU_STORE_ALPHAS)
    assert store_pairs(case) == [65536] * len(EMU_STORE_ALPHAS)
    got, want, routes = cc.run_case(emu, EmuMem(), case, None, log=emu)
    assert form in cc.route_log(emu, case), form
    cc.check_bytes(got, want, form)
    assert routes == ["blend"] + ["fused"] * len(EMU_STORE_ALPHAS), routes
