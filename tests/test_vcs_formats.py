"""What the library makes of each video format, without a GPU: the emulated library (tests/cudaemu) against the fixture
tests/golden/vcs_formats.json (tests/golden/make_vcs_formats.py).  It pins b200_video_info_set_format and
b200_video_info_size for every format, the b200_vcs_create status of every format pair over sizes, plane layouts,
colorimetry and destination rectangles, the plans' introspection and the bytes of emulated converts."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import make_vcs_formats as mf  # noqa: E402

pytestmark = pytest.mark.timeout(600)


@pytest.fixture(scope="module")
def emu():
    return mf.load()


@pytest.fixture(scope="module")
def want():
    return json.load(open(mf.FIXTURE))


def differing(got, want):
    return sorted(k for k in set(got) | set(want) if got.get(k) != want.get(k))


def test_grid_matches_fixture(want):
    assert json.loads(json.dumps({"formats": mf.FMT, "unknown": mf.UNKNOWN, "info_sizes": mf.INFO_SIZES,
                                  "create_sizes": mf.CREATE_SIZES, "colorimetry": mf.COLORIMETRY,
                                  "convert_sizes": mf.CONVERT_SIZES, "borders": mf.BORDERS,
                                  "status": mf.STATUS})) == want["grid"]


def test_video_info(emu, want):
    got = json.loads(json.dumps(mf.record_info(*emu)))
    assert not differing(got, want["info"]), differing(got, want["info"])


@pytest.mark.parametrize("fi", list(mf.FMT))
def test_create_status_and_plans(emu, want, fi):
    status, plans = mf.record_pairs(*emu, fi)
    mine = lambda d: {k: v for k, v in d.items() if k.startswith(fi + ">")}   # noqa: E731
    bad = differing(status, mine(want["status"]))
    assert not bad, "status differs for %s: got %s, want %s" % (bad, status.get(bad[0]), want["status"].get(bad[0]))
    bad = differing(plans, mine(want["plans"]))
    assert not bad, "introspection differs for %s" % bad


@pytest.mark.parametrize("fi", list(mf.FMT))
def test_convert_bytes(emu, want, fi):
    got = mf.record_bytes(*emu, fi)
    bad = differing(got, {k: v for k, v in want["bytes"].items() if k.startswith(fi + ">")})
    assert not bad, "output bytes differ for %s" % bad
