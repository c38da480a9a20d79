"""The fused route's plane scalers on the device (tests/comp_fused_cases.py): every row's conversion on worst-case content
of its own taps at clipped positions and alphas copy / 254 / 128 / 1, and comp_store's full (p, v, a) domain - every
alpha 1 .. 255 and copy - through two byte-picking forms, against oracle_vcs_convert + oracle_compositor_yuv.
tests/test_comp_fused.py asserts from the emulated launch log which form each row launches."""
import pytest

import comp_convert_cases as cc
import comp_domain as cd
import comp_fused_cases as cf
from test_comp_convert_gpu import run

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib(cuda_device):
    from gstreamer_b200._lib import lib
    return lib


@pytest.mark.parametrize("row", cf.ROWS, ids=lambda r: f"{r.out}-{r.form}")
def test_row(lib, row):
    got, want, routes = run(lib, cf.row_case(row))
    cc.check_bytes(got, want, row.form)
    assert set(routes) == {"fused"}, routes


@pytest.mark.parametrize("form", list(cf.STORE_FORMS))
def test_store_domain(lib, form):
    alphas = [cd.alpha_for(k, 255) for k in range(1, 256)] + [1.0]
    for part in cd.chunks(alphas, cd.MAX_PADS - 1):
        got, want, routes = run(lib, cf.store_case(form, part))
        cc.check_bytes(got, want, f"{form} alphas {part[0]} ..")
        assert routes == ["blend"] + ["fused"] * len(part), routes
