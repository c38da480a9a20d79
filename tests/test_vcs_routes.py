"""Which kernels a convert launches, per handle configuration, without a GPU: the emulated library (tests/cudaemu) logs
every launch of b200_vcs_convert.  The fixture tests/golden/vcs_routes.json (tests/golden/make_vcs_routes.py) pins the
launch sequences, status codes and what the handle reports about them (plan_info.kernel_variant, n_launches_per_convert,
kernel_name) over the element's format pairs, chroma sitings, sizes reaching every route, all methods, destination
rectangles, forced variants, frame alignments and the A/B knobs."""
import json
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import make_vcs_routes as mr  # noqa: E402

pytestmark = pytest.mark.timeout(600)

# every kernel a convert launches (tests/vcs_batch_cases.py runs each of them on batches of distinct frames)
GRID_KERNELS = {"vcs_border_kernel", "vcs_down420_kernel", "vcs_generic_kernel", "vcs_l2mma_kernel", "vcs_lanczos2_kernel",
                "vcs_lanczos2_v2_kernel", "vcs_light_kernel", "vcs_ntap_kernel", "vcs_ntap_vfirst_kernel", "vcs_planes_fast_kernel",
                "vcs_planes_fast_vfirst_kernel", "vcs_planes_kernel", "vcs_planes_vec_kernel", "vcs_rgb2ayuv_kernel",
                "vcs_rgb420_kernel", "vcs_rgb_deinterleave_kernel", "vcs_yuy2_420_kernel", "vcs_yuy2_ayuv_kernel"}

# kernel_name -> the launched kernels it stands for: the n-tap launcher picks its vertical-first form where that is
# cheaper, the plane launcher runs copy / halve planes through vcs_planes_vec_kernel
NAMED = {"vcs_ntap_kernel": {"vcs_ntap_kernel", "vcs_ntap_vfirst_kernel"},
         "vcs_planes_kernel": {"vcs_planes_kernel", "vcs_planes_vec_kernel"}}


@pytest.fixture(scope="module")
def routes():
    return json.loads(json.dumps(mr.record())), json.load(open(mr.FIXTURE))


@pytest.mark.parametrize("knob", [None] + mr.KNOBS)
def test_routes_match_fixture(routes, knob):
    got, want = routes
    assert got["grid"] == want["grid"]
    g, w = mr.expand(got, knob), mr.expand(want, knob)
    assert g.keys() == w.keys()
    bad = [(k, m) for k in w for m in range(len(w[k])) if g[k][m] != w[k][m]]
    assert not bad, "%d of %d handle records differ, first %s: got %s, want %s" % (
        len(bad), 10 * len(w), bad[0], g[bad[0][0]][bad[0][1]], w[bad[0][0]][bad[0][1]])


def test_grid_reaches_every_kernel(routes):
    got, _ = routes
    launched = {re.sub(r"<.*", "", x) for x in got["launches"] for x in x}
    assert launched == GRID_KERNELS


@pytest.mark.parametrize("knob", [None] + mr.KNOBS)
def test_introspection_describes_aligned_launches(routes, knob):
    """on 16-byte aligned frames: n_launches_per_convert counts the launches, kernel_name names one of them (NAMED).
    B200_CROSS_GENERIC swaps the chain's first launch for the generic kernel and leaves the name: not name-checked."""
    got, _ = routes
    checked = 0
    for key, results in mr.expand(got, knob).items():
        for m, r in enumerate(results):
            for s in r[1:]:
                if not s[5]:
                    continue
                st, launches = s[5][0]
                assert st == 0, (key, m, s)
                assert s[3] == len(launches), (key, m, s)
                if knob != "B200_CROSS_GENERIC=1":
                    names = {re.sub(r"<.*", "", x) for x in launches}
                    assert NAMED.get(s[4], {s[4]}) & names, (key, m, s)
                checked += 1
    assert checked > (10000 if knob is None else 500)
