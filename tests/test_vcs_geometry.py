"""The launch geometry of every tiled kernel, without a GPU: the emulated library (tests/cudaemu) logs each launch of
b200_vcs_convert with its grid, block and dynamic shared-memory bytes.  The fixture tests/golden/vcs_geometry.json
(tests/golden/make_vcs_geometry.py) pins them, with get_plan_info's tile_w, tile_h and smem_bytes, over the converter's
format pairs, sizes and methods, production sizes, and each tile-shape override, as one digest per format pair."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import make_vcs_geometry as mg  # noqa: E402

pytestmark = pytest.mark.timeout(900)


@pytest.fixture(scope="module")
def geometry():
    return json.loads(json.dumps(mg.record())), json.load(open(mg.FIXTURE))


@pytest.mark.parametrize("part,knob", [("cases", None), ("prod", None)] + [("knobs", k) for k in mg.KNOBS])
def test_geometry_matches_fixture(geometry, part, knob):
    got, want = geometry
    assert got["grid"] == want["grid"]
    g, w = (got[part], want[part]) if knob is None else (got[part][knob], want[part][knob])
    assert g.keys() == w.keys()
    bad = [p for p in w if g[p] != w[p]]
    assert not bad, "%d of %d format pairs differ: %s (make_vcs_geometry.py --dump PAIR lists a pair's records)" % (
        len(bad), len(w), bad)


def test_knobs_change_the_shape(geometry):
    """each override selects a shape the search does not: some production record differs from the default's"""
    got, _ = geometry
    for k in mg.KNOBS:
        assert got["knobs"][k] != got["prod"], k
