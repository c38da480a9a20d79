"""The compositor's kernels on the device over their input domains, against the integer model of tests/comp_domain.py
(which tests/test_comp_domain.py pins against the oracle and the reference build).  The expected values are the model
evaluated in torch int64 on the device.

Beyond the CPU file's domains: OVERLAY / OVERLAY_ADD colours over the full (s, d, as, dalpha) domain at pad alpha 1.0
for both alpha positions (about 1.43 G pixels each, in chunks), the 10-bit blend over all in-range (s, d) at all 1022
blend alphas, the 16-bit blend at all 65534 blend alphas over 1024 structured (s, d) pairs, every alpha edge at every
range through all three entry points.  This is where the kernels' PTX (cvt.pack.sat in sat_pack2) is checked; the
emulated build has plain C in its place.
"""
import numpy as np
import pytest

import comp_convert_cases as cc
import comp_domain as cd
from test_comp_domain import (EDGE_SETS, EDGE_YUV, GRID, RGB_CHUNK, YUV_CHUNK, alpha_domain, blend_domain, edge_calls_rgb,
                              edge_calls_yuv, plane_domain, run_rgb_chunk, run_too_many_pads, run_yuv_chunk, structured,
                              wide_alphas)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cd.Device()


def dcheck(got, want, what):
    import torch
    if not torch.equal(got, want):
        bad = torch.nonzero(got != want)
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} values differ, first at {list(i)}: got {int(got[i])} want {int(want[i])}")


def rgb_case(dev, fmt, bg, d, s, bands, entry="blend"):
    d, s = dev.asarray(d), dev.asarray(s)
    dcheck(cd.rgb_pads(dev, fmt, bg, d, s, bands, entry=entry), cd.rgb_expected(fmt, bg, d, s, bands), f"{fmt} {bands[0]}")


def yuv_case(dev, name, d, s, bands, entry="yuv"):
    d, s = dev.asarray(d), dev.asarray(s)
    dcheck(cd.yuv_pads(dev, name, d, s, bands, entry), cd.yuv_expected(cd.YUV[name][1], d, s, bands), f"{name} {bands[0]}")


# ---- the CPU file's domains -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", list(cd.RGB))
def test_blend_all(dev, fmt):
    d, s = blend_domain(fmt, range(256))
    rgb_case(dev, fmt, cd.BLACK, d, s, [(0, 256, 1.0, cd.OVER)])


@pytest.mark.parametrize("fmt", list(cd.RGB))
@pytest.mark.parametrize("op", [cd.SOURCE, cd.OVER])
def test_pad_alpha_product_all(dev, fmt, op):
    for part in cd.chunks(list(range(1, 256)), cd.MAX_PADS - 1):
        d, s = alpha_domain(fmt, part, rows=4)
        rgb_case(dev, fmt, cd.WHITE, d, s, cd.bands_of([cd.alpha_for(k, 255) for k in part], 4, op))


@pytest.mark.parametrize("fmt", list(cd.RGB))
@pytest.mark.parametrize("op", [cd.OVER, cd.ADD], ids=["overlay", "overlay_add"])
def test_overlay_alpha_byte_all(dev, fmt, op):
    for part in cd.chunks(list(range(1, 256)), cd.MAX_PADS - 1):
        d, s = alpha_domain(fmt, part)
        rgb_case(dev, fmt, cd.TRANSPARENT, d, s, cd.bands_of([cd.alpha_for(k, 255) for k in part], 256, op))


@pytest.mark.parametrize("fmt", ["BGRA", "ARGB"])
@pytest.mark.parametrize("op", [cd.OVER, cd.ADD], ids=["overlay", "overlay_add"])
def test_overlay_colour_grid(dev, fmt, op):
    d, s = blend_domain(fmt, GRID, GRID)
    rgb_case(dev, fmt, cd.TRANSPARENT, d, s, [(0, d.shape[0], 1.0, op)])


def test_u8_all(dev):
    for part in cd.chunks(list(range(1, 256)), cd.MAX_PADS - 1):
        d, s, rows = plane_domain(8, 1 << 16, len(part))
        yuv_case(dev, "Y444", d, s, cd.bands_of([cd.alpha_for(k, 255) for k in part], rows, cd.OVER))


@pytest.mark.parametrize("name", ["Y444_12LE", "Y444_16LE"])
def test_wide_in_range(dev, name):
    nbits = cd.YUV[name][1]
    for part in cd.chunks(wide_alphas(nbits), 12):
        d, s, rows = plane_domain(nbits, 1 << 20, len(part), structured(nbits))
        yuv_case(dev, name, d, s, cd.bands_of([cd.alpha_for(k, (1 << nbits) - 1) for k in part], rows, cd.OVER))


@pytest.mark.parametrize("name", ["Y444_10LE", "Y444_12LE", "Y444_16LE"])
def test_wide_out_of_range(dev, name):
    nbits = cd.YUV[name][1]
    values = structured(nbits, 512, full=True)
    ks = wide_alphas(nbits, 40, seed=4)
    for part in cd.chunks(ks, cd.MAX_PADS - 1):
        d, s, rows = plane_domain(nbits, len(values) ** 2, len(part), values)
        yuv_case(dev, name, d, s, cd.bands_of([cd.alpha_for(k, (1 << nbits) - 1) for k in part], rows, cd.OVER))


# ---- full domains ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["BGRA", "ARGB"])
@pytest.mark.parametrize("op", [cd.OVER, cd.ADD], ids=["overlay", "overlay_add"])
def test_overlay_colour_full(dev, fmt, op):
    """all (s, d, as, dalpha) at pad alpha 1.0 on a transparent background: rows are the (as, dalpha) pairs, the three
    colour bytes of a row's 21846 pixels carry all 65536 (s, d) pairs; 8 source alphas per call"""
    import torch
    ai = cd.RGB[fmt][1]
    ci = [c for c in range(4) if c != ai]
    W, per = 21846, 8
    q = torch.arange(3 * W, device="cuda") % 65536
    sc, dc = (q & 255).to(torch.uint8).view(W, 3), (q >> 8).to(torch.uint8).view(W, 3)
    for as0 in range(0, 256, per):
        H = per * 256
        r = torch.arange(H, device="cuda")
        s = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
        d = torch.empty_like(s)
        s[:, :, ci] = sc
        d[:, :, ci] = dc
        s[:, :, ai] = (as0 + r // 256).to(torch.uint8)[:, None]
        d[:, :, ai] = (r % 256).to(torch.uint8)[:, None]
        bands = [(0, H, 1.0, op)]
        dcheck(cd.rgb_pads(dev, fmt, cd.TRANSPARENT, d, s, bands), cd.rgb_expected(fmt, cd.TRANSPARENT, d, s, bands),
               f"{fmt} as {as0} .. {as0 + per - 1}")


def wide_sweep(dev, name, ks, values, per_call):
    """the wide blend at every integer alpha of ks over all pairs of `values`; the model evaluated at once per call with
    the alpha of each row"""
    import torch
    nbits = cd.YUV[name][1]
    r = (1 << nbits) - 1
    n_pairs = len(values) ** 2
    for part in cd.chunks(list(ks), per_call):
        d, s, rows = plane_domain(nbits, n_pairs, len(part), values)
        d, s = dev.asarray(d), dev.asarray(s)
        bands = cd.bands_of([cd.alpha_for(k, r) for k in part], rows, cd.OVER)
        got = cd.yuv_pads(dev, name, d, s, bands)
        a = torch.tensor(part, device="cuda").repeat_interleave(rows)[None, :, None]
        dcheck(got, cd.blend_wide(s.long(), d.long(), a, nbits).to(torch.int32), f"{name} alphas {part[0]} .. {part[-1]}")


def test_u10_all_alphas(dev):
    """all in-range (s, d) at every blend alpha 1 .. 1022"""
    wide_sweep(dev, "Y444_10LE", range(1, 1023), list(range(1024)), 16)


def test_u16_all_alphas(dev):
    """1024 structured (s, d) pairs (32 x 32 values: the ends, powers of two and their neighbours) at every blend
    alpha 1 .. 65534"""
    v = structured(16, 32)
    values = [v[i] for i in np.linspace(0, len(v) - 1, 32).round().astype(int)]
    assert len(set(values)) == 32 and values[0] == 0 and values[-1] == 65535
    wide_sweep(dev, "Y444_16LE", range(1, 65535), values, cd.MAX_PADS - 1)


# ---- alpha edges, chunks, the pad limit -----------------------------------------------------------------------------------
@pytest.mark.parametrize("entry", ["blend", "convert"])
def test_alpha_edges(dev, entry):
    """every k / range and both its neighbours (a sample of 65535), RGB and planar outputs, alphas above 1.0 included"""
    for fmt in ("BGRA", "ARGB"):
        for d, s, bands, bg in edge_calls_rgb(cd.alpha_edges(255), fmt):
            rgb_case(dev, fmt, bg, d, s, bands, entry)
    assert EDGE_SETS[1023] is None and EDGE_SETS[4095] is None
    for rng, name in EDGE_YUV:
        for d, s, bands in edge_calls_yuv(rng, cd.YUV[name][1]):
            yuv_case(dev, name, d, s, bands, "yuv" if entry == "blend" else "convert")


@pytest.mark.parametrize("n,W", RGB_CHUNK)
@pytest.mark.parametrize("entry", ["blend", "convert"])
def test_rgb_chunks(dev, n, W, entry):
    run_rgb_chunk(dev, n, W, entry)


@pytest.mark.parametrize("n,name", YUV_CHUNK)
@pytest.mark.parametrize("entry", ["yuv", "convert"])
def test_yuv_chunks(dev, n, name, entry):
    run_yuv_chunk(dev, n, name, entry)


def test_too_many_pads(dev):
    run_too_many_pads(dev)


@pytest.mark.parametrize("out_name", ["NV12", "I420", "BGRA"])
def test_convert_64_pads_mixed_routes(dev, out_name):
    """b200_comp_blend_convert with 64 pads: converted (fused or two-pass) and blend-kernel pads interleaved, across the
    launch chunks of both blend kernels"""
    from test_comp_convert_gpu import run
    rng = np.random.default_rng(64 + cc.FMT[out_name])
    case = cc.random_case(rng, out_name, 1, max_size=(80, 48), max_pads=64, min_pads=64, pad_max=(24, 16))
    got, want, routes = run(dev.lib, case)
    cc.check_bytes(got, want, f"{out_name} 64 pads")
    assert len(routes) == 64
    assert {"blend", "two-pass"} <= set(routes), routes
    if out_name != "BGRA":
        assert "fused" in routes, routes
