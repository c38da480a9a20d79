"""Which kernels an audio resampler call launches, per handle configuration, without a GPU: the emulated library
(tests/cudaemu) logs every launch of b200_ars_process with its grid, block and dynamic shared-memory bytes.  The fixture
tests/golden/ars_routes.json (tests/golden/make_ars_routes.py) pins the launches, status codes, output frame counts and
plan_info over the sample formats, resample methods and filter modes, rate pairs reaching every route, channel counts,
pointer alignments, a rate update and the audio knobs."""
import json
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import make_ars_routes as mr  # noqa: E402

pytestmark = pytest.mark.timeout(600)


@pytest.fixture(scope="module")
def routes():
    return json.loads(json.dumps(mr.record())), json.load(open(mr.FIXTURE))


def kernels(launches):
    return [re.sub(r" grid=.*", "", x) for x in launches]


def calls_of(result):
    return [c for seq in result[2::2] for c in seq]


@pytest.mark.parametrize("knob", [None] + mr.KNOBS)
def test_routes_match_fixture(routes, knob):
    got, want = routes
    assert got["grid"] == want["grid"]
    g, w = mr.expand(got, knob), mr.expand(want, knob)
    assert g.keys() == w.keys()
    bad = [k for k in w if g[k] != w[k]]
    assert not bad, "%d of %d handle records differ, first %s: got %s, want %s" % (len(bad), len(w), bad[0], g[bad[0]], w[bad[0]])


def test_grid_reaches_every_kernel(routes):
    got, _ = routes
    launched = set(kernels(got["launches"]))
    assert launched == {"ars_small_kernel<0>", "ars_small_kernel<1>", "ars_small_kernel<2>", "ars_small_kernel<3>",
                        "ars_pipe_kernel", "ars_pipe_kernel_v1", "ars_pipe_kernel_s16",
                        "ars_tile_kernel<128, 4>", "ars_tile_kernel<128, 2>", "ars_tile_kernel<128, 1>",
                        "ars_tile_kernel<64, 2>", "ars_tile_kernel<64, 1>", "ars_tile_kernel<32, 1>",
                        "ars_tile_kernel_s16<128>", "ars_tile_kernel_s16<64>", "ars_full_kernel",
                        "ars_interp_kernel<true>", "ars_interp_kernel<false>",
                        "ars_direct_kernel<1, true>", "ars_direct_kernel<1, false>", "ars_direct_kernel<2, true>",
                        "ars_direct_kernel<2, false>", "ars_direct_kernel<3, true>", "ars_direct_kernel<3, false>",
                        "ars_history_kernel", "ars_history_kernel_x<unsigned short>", "ars_history_kernel_x<unsigned long long>"}
    refused = [c for r in mr.expand(got).values() if len(r) > 1 for c in calls_of(r) if c[0] != 0]
    assert refused and all(c[0] == -2 and not c[2] for c in refused)          # B200_ERR_UNSUPPORTED, nothing launched


def first_kernels(got, key):
    """the resampling kernel of each call of one record that produced output, before the update"""
    return {kernels(c[2])[0] for c in mr.expand(got)[key][2] if c[1]}


def test_named_routes(routes):
    """the routes other tests name: 1480 taps take the generic F32 kernel; whole 128-channel blocks at 16-byte alignment the
    persistent pipelines"""
    got, _ = routes
    assert first_kernels(got, "F32 kaiser-auto-cubic 96000>8000 q7 1ch") == {"ars_full_kernel"}
    for fmt, pipe in (("F32", "ars_pipe_kernel"), ("S16", "ars_pipe_kernel_s16")):
        for ch in (128, 256):
            for rates in ("48000>44100", "44100>48000"):
                r = mr.expand(got)["%s kaiser-auto-cubic %s q4 %dch" % (fmt, rates, ch)]
                aligned = [c for c, (n, a) in zip(r[2], mr.calls(fmt)[0]) if a == 16 and c[1]]
                assert aligned and all(kernels(c[2])[0] == pipe for c in aligned), (fmt, ch, rates)
