"""The compositor's pixel arithmetic over its input domain, without a GPU (tests/comp_domain.py).

  model == oracle     every operator of the packed RGB and planar compositors over whole domains: BLEND over all
                      (s, d, as), SOURCE and the pad-alpha product over all (as, alpha), OVERLAY / OVERLAY_ADD colours over
                      all (s, d) on an (as, dalpha) grid and their alpha byte over all (as, dalpha, alpha), the 8-bit plane
                      blend over all (s, d, a), the 10 / 12 / 16-bit blends over in-range and out-of-range samples;
  oracle == reference the same domains (the rows the `ref` tests sample) through the reference build;
  alpha edges         the quantisation of the pad alpha at every k / range and both its neighbours, through the oracle
                      and through b200_comp_blend, b200_comp_blend_yuv and b200_comp_blend_convert of the emulated library;
  emulated == model   the kernels themselves (tests/cudaemu) on reduced domains.

The emulated build replaces the kernels' one PTX instruction (cvt.pack.sat in sat_pack2) with plain C, so only
tests/test_comp_domain_gpu.py checks the real instruction; here the kernels' integer paths (div255 on 16-bit lanes, the
reciprocal table, the byte selectors of each alpha position, the wrapping wide blend) are what is checked.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cudaemu"))

import comp_domain as cd  # noqa: E402
from oracle import bindings as ob  # noqa: E402

pytestmark = pytest.mark.timeout(900)


# ---- the oracle and the reference on domain frames ------------------------------------------------------------------------
def _lib_fn(which, name):
    return getattr(ob.oracle(), "oracle_" + name) if which == "oracle" else getattr(ob.ref(), "ref_" + name)


def checker_rgb(which, fmt, bg, d, s, bands):
    """the oracle's (or the reference's) output of the domain call rgb_pads describes"""
    H, W = d.shape[:2]
    pads = (ob.OraclePad * (1 + len(bands)))()
    keep = [np.ascontiguousarray(d)]
    pads[0].data, pads[0].width, pads[0].height, pads[0].stride = keep[0].ctypes.data, W, H, W * 4
    pads[0].xpos, pads[0].ypos, pads[0].alpha, pads[0].op = 0, 0, 1.0, cd.SOURCE
    for i, (y0, y1, alpha, op) in enumerate(bands, 1):
        keep.append(np.ascontiguousarray(s[y0:y1]))
        pads[i].data, pads[i].width, pads[i].height, pads[i].stride = keep[-1].ctypes.data, W, y1 - y0, W * 4
        pads[i].xpos, pads[i].ypos, pads[i].alpha, pads[i].op = 0, y0, alpha, op
    out = np.full((H, W, 4), 0x33, np.uint8)
    _lib_fn(which, "compositor")(cd.RGB[fmt][0], out.ctypes.data, W, H, W * 4, bg, pads, len(pads))
    return out


def checker_yuv(which, name, d, s, bands):
    fmt, nbits = cd.YUV[name]
    H, W = d.shape[1:]
    pads = (ob.OraclePad * (1 + len(bands)))()
    keep = [np.ascontiguousarray(cd.yuv_planes_to_bytes(d, nbits))]
    pads[0].data, pads[0].width, pads[0].height, pads[0].stride = keep[0].ctypes.data, W, H, 0
    pads[0].xpos, pads[0].ypos, pads[0].alpha, pads[0].op = 0, 0, 1.0, cd.SOURCE
    for i, (y0, y1, alpha, op) in enumerate(bands, 1):
        keep.append(np.ascontiguousarray(cd.yuv_planes_to_bytes(np.ascontiguousarray(s[:, y0:y1]), nbits)))
        pads[i].data, pads[i].width, pads[i].height, pads[i].stride = keep[-1].ctypes.data, W, y1 - y0, 0
        pads[i].xpos, pads[i].ypos, pads[i].alpha, pads[i].op = 0, y0, alpha, op
    out = np.zeros(W * H * 3 * (1 if nbits == 8 else 2), np.uint8)
    assert _lib_fn(which, "compositor_yuv")(fmt, out.ctypes.data, W, H, cd.BLACK, 1, pads, len(pads)) == 0
    return cd.yuv_bytes_to_planes(out, nbits, (3, H, W))


def check(got, want, what):
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        raise AssertionError(f"{what}: {len(bad)} values differ, first at {bad[0].tolist()}: got {got[tuple(bad[0])]} "
                             f"want {want[tuple(bad[0])]}")


# ---- domain frames (numpy; tests/test_comp_domain_gpu.py builds the same on the device) -----------------------------------
def blend_domain(fmt, as_values, da=None):
    """rows: one per (as, dalpha) in as_values x da (dalpha: (as * 37) & 255 when da is None, which BLEND ignores);
    columns: 21846 pixels whose three colour bytes carry all 65536 (s, d) pairs"""
    ai = cd.RGB[fmt][1]
    ci = [c for c in range(4) if c != ai]
    W = 21846
    s_c, d_c = cd.pair_grid(3 * W)
    rows = [(a, (a * 37) & 255 if da is None else b) for a in as_values for b in (da if da is not None else [None])]
    H = len(rows)
    s, d = np.zeros((H, W, 4), np.uint8), np.zeros((H, W, 4), np.uint8)
    s[:, :, ci] = s_c.reshape(W, 3)
    d[:, :, ci] = d_c.reshape(W, 3)
    s[:, :, ai] = np.array([r[0] for r in rows], np.uint8)[:, None]
    d[:, :, ai] = np.array([r[1] for r in rows], np.uint8)[:, None]
    return d, s


def alpha_domain(fmt, ks, rows=256, seed=0):
    """bands of `rows` rows, one per pad alpha k: source alpha byte = column (0 .. 255), destination alpha byte = row, colours
    at the corners (0 / 255, by pixel position) - every (as, dalpha) under every pad alpha"""
    ai = cd.RGB[fmt][1]
    H, W = rows * len(ks), 256
    y, x = np.mgrid[0:H, 0:W]
    s, d = np.zeros((H, W, 4), np.uint8), np.zeros((H, W, 4), np.uint8)
    for j, c in enumerate(c for c in range(4) if c != ai):
        s[..., c] = 255 * ((x + y + j) & 1)
        d[..., c] = 255 * (((x >> 1) + j) & 1)
    s[..., ai] = x
    d[..., ai] = y % rows
    return d, s


def plane_domain(nbits, n_pairs, n_bands, values=None):
    """[3, rows * n_bands, W] samples: each band carries the (s, d) pairs of `values` x `values` (all in-range values
    when None) across its three planes"""
    if values is None:
        values = np.arange(1 << nbits, dtype=np.int64)
    values = np.asarray(values, np.int64)
    nv = len(values)
    q = np.arange(n_pairs, dtype=np.int64) % (nv * nv)
    sv, dv = values[q % nv], values[q // nv]
    W = 256 if n_pairs < 1 << 20 else 1024
    rows = -(-n_pairs // (3 * W))
    dt = np.uint8 if nbits == 8 else np.int32
    s = np.zeros((3, rows, W), dt)
    d = np.zeros((3, rows, W), dt)
    s.reshape(-1)[:n_pairs], d.reshape(-1)[:n_pairs] = sv, dv
    return np.tile(d, (1, n_bands, 1)), np.tile(s, (1, n_bands, 1)), rows


def structured(nbits, n=1024, full=False):
    """n sample values of an n-bit plane: both ends, the middle, powers of two and their neighbours, the rest evenly
    spread; full=True spreads them over the whole 16-bit range (samples above 2^n - 1 included)"""
    top = 65535 if full else (1 << nbits) - 1
    v = {0, 1, 2, top - 1, top, (1 << nbits) - 2, (1 << nbits) - 1, 1 << (nbits - 1)}
    for b in range(16 if full else nbits):
        v |= {(1 << b) - 1, 1 << b, (1 << b) + 1}
    v = {x for x in v if 0 <= x <= top}
    v |= set(np.linspace(0, top, max(0, n - len(v))).astype(np.int64).tolist())
    return sorted(v)


def wide_alphas(nbits, n=20, seed=0):
    """at least 16 integer alphas of an n-bit blend: the edges (1, 2, 3, the middle, range - 2, range - 1, range - reached
    only by a pad alpha above 1.0) and random ones"""
    r = (1 << nbits) - 1
    ks = {1, 2, 3, r // 2, r // 2 + 1, r - 2, r - 1, r}
    ks |= set(np.random.default_rng(seed).integers(1, r, n).tolist())
    return sorted(ks)


# ---- model == oracle ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["BGRA", "ARGB"])
def test_blend_all(fmt):
    """BLEND at pad alpha 1.0 over all (s, d, as): 2^24 colour bytes"""
    d, s = blend_domain(fmt, range(256))
    bands = [(0, 256, 1.0, cd.OVER)]
    check(checker_rgb("oracle", fmt, cd.BLACK, d, s, bands), cd.rgb_expected(fmt, cd.BLACK, d, s, bands), fmt)


@pytest.mark.parametrize("fmt", ["RGBA", "ABGR"])
@pytest.mark.parametrize("op", [cd.SOURCE, cd.OVER])
def test_pad_alpha_product_all(fmt, op):
    """SOURCE (alpha byte floor(as * k / 255)) and BLEND at every integer pad alpha k over every as: all (as, alpha)"""
    ks = list(range(1, 256))
    for part in cd.chunks(ks, cd.MAX_PADS - 1):
        d, s = alpha_domain(fmt, part, rows=4)
        bands = cd.bands_of([cd.alpha_for(k, 255) for k in part], 4, op)
        check(checker_rgb("oracle", fmt, cd.WHITE, d, s, bands), cd.rgb_expected(fmt, cd.WHITE, d, s, bands), f"{fmt} {part[0]}")


GRID = sorted({0, 1, 2, 127, 128, 254, 255} | set(range(0, 256, 17)))


@pytest.mark.parametrize("op", [cd.OVER, cd.ADD], ids=["overlay", "overlay_add"])
@pytest.mark.parametrize("fmt", ["BGRA", "ARGB"])
def test_overlay_colour_grid(fmt, op):
    """OVERLAY / OVERLAY_ADD colours over all (s, d) x the (as, dalpha) grid (0, 1, 2, 127, 128, 254, 255, every 17th)"""
    d, s = blend_domain(fmt, GRID, GRID)
    bands = [(0, d.shape[0], 1.0, op)]
    check(checker_rgb("oracle", fmt, cd.TRANSPARENT, d, s, bands), cd.rgb_expected(fmt, cd.TRANSPARENT, d, s, bands), fmt)


@pytest.mark.parametrize("op", [cd.OVER, cd.ADD], ids=["overlay", "overlay_add"])
def test_overlay_alpha_byte_all(op):
    """the alpha byte (and the corner colours) of OVERLAY / OVERLAY_ADD over all (as, dalpha, pad alpha): 2^24"""
    for fmt in ("BGRA", "ABGR"):
        for part in cd.chunks(list(range(1, 256)), cd.MAX_PADS - 1):
            d, s = alpha_domain(fmt, part)
            bands = cd.bands_of([cd.alpha_for(k, 255) for k in part], 256, op)
            check(checker_rgb("oracle", fmt, cd.TRANSPARENT, d, s, bands), cd.rgb_expected(fmt, cd.TRANSPARENT, d, s, bands),
                  f"{fmt} {part[0]}")


def test_u8_all():
    """the 8-bit plane blend over all (s, d, a), a = 1 .. 255 (255 only from a pad alpha above 1.0)"""
    for part in cd.chunks(list(range(1, 256)), cd.MAX_PADS - 1):
        d, s, rows = plane_domain(8, 1 << 16, len(part))
        bands = cd.bands_of([cd.alpha_for(k, 255) for k in part], rows, cd.OVER)
        check(checker_yuv("oracle", "Y444", d, s, bands), cd.yuv_expected(8, d, s, bands), f"u8 {part[0]}")


@pytest.mark.parametrize("name", ["Y444_10LE", "Y444_12LE", "Y444_16LE"])
def test_wide_in_range(name):
    """10 / 12 / 16-bit blends: in-range (s, d) - all of them at 10 bits, 1024 x 1024 structured values above - at 16 or
    more alphas, the edges included"""
    nbits = cd.YUV[name][1]
    values = None if nbits == 10 else structured(nbits)
    ks = wide_alphas(nbits)
    assert len(ks) >= 16
    for part in cd.chunks(ks, 12):
        d, s, rows = plane_domain(nbits, 1 << 20, len(part), values)
        bands = cd.bands_of([cd.alpha_for(k, (1 << nbits) - 1) for k in part], rows, cd.OVER)
        check(checker_yuv("oracle", name, d, s, bands), cd.yuv_expected(nbits, d, s, bands), f"{name} {part}")


@pytest.mark.parametrize("name", ["Y444_10LE", "Y444_12LE", "Y444_16LE"])
def test_wide_out_of_range(name):
    """samples anywhere in the 16-bit range: the wrapping statement carries them through.  d*(2^n - a) + s*a never passes
    65535 * 2^n < 2^32, so nothing wraps and the 16-bit clamp never fires - the clamped and unclamped statements agree
    over the whole domain, and results above 2^n - 1 come out as they are"""
    nbits = cd.YUV[name][1]
    r = (1 << nbits) - 1
    values = structured(nbits, 512, full=True)
    ks = wide_alphas(nbits, 8, seed=1)
    d, s, rows = plane_domain(nbits, len(values) ** 2, len(ks), values)
    bands = cd.bands_of([cd.alpha_for(k, r) for k in ks], rows, cd.OVER)
    want = cd.yuv_expected(nbits, d, s, bands)
    check(checker_yuv("oracle", name, d, s, bands), want, name)
    assert nbits == 16 or want.max() > r
    v = np.array(values, np.int64)
    for k in range(1, r + 1, max(1, r // 4096)):       # the clamp is a no-op for every alpha at the extremes
        for sv, dv in ((v, 65535), (65535, v), (v, 0), (0, v), (v, v[::-1])):
            u = cd.blend_wide_unclamped(np.asarray(sv), np.asarray(dv), k, nbits)
            assert u.max() <= 65535 and u.min() >= 0


# ---- oracle == reference --------------------------------------------------------------------------------------------------
@pytest.mark.ref
@pytest.mark.parametrize("fmt", ["BGRA", "ARGB"])
def test_ref_rgb(fmt):
    """the reference build's bytes on the RGB domains (as rows sampled every 5th)"""
    d, s = blend_domain(fmt, range(0, 256, 5))
    bands = [(0, d.shape[0], 1.0, cd.OVER)]
    check(checker_rgb("ref", fmt, cd.BLACK, d, s, bands), checker_rgb("oracle", fmt, cd.BLACK, d, s, bands), "blend")
    d, s = blend_domain(fmt, GRID[::2], GRID[::2])
    for op in (cd.OVER, cd.ADD):
        bands = [(0, d.shape[0], 1.0, op)]
        check(checker_rgb("ref", fmt, cd.TRANSPARENT, d, s, bands), checker_rgb("oracle", fmt, cd.TRANSPARENT, d, s, bands),
              f"overlay {op}")
    for op, bg in ((cd.SOURCE, cd.WHITE), (cd.OVER, cd.WHITE), (cd.OVER, cd.TRANSPARENT), (cd.ADD, cd.TRANSPARENT)):
        for part in cd.chunks(list(range(1, 256)), cd.MAX_PADS - 1):
            d, s = alpha_domain(fmt, part, rows=8)
            bands = cd.bands_of([cd.alpha_for(k, 255) for k in part], 8, op)
            check(checker_rgb("ref", fmt, bg, d, s, bands), checker_rgb("oracle", fmt, bg, d, s, bands), f"alpha {op} {bg}")


@pytest.mark.ref
@pytest.mark.parametrize("name", list(cd.YUV))
def test_ref_planes(name):
    nbits = cd.YUV[name][1]
    r = (1 << nbits) - 1
    if nbits == 8:
        ks, values = list(range(1, 256, 3)), None
    else:
        ks, values = wide_alphas(nbits, 8, seed=2), structured(nbits, 256, full=True)
    for part in cd.chunks(ks, cd.MAX_PADS - 1):
        d, s, rows = plane_domain(nbits, 1 << 16, len(part), values)
        bands = cd.bands_of([cd.alpha_for(k, r) for k in part], rows, cd.OVER)
        check(checker_yuv("ref", name, d, s, bands), checker_yuv("oracle", name, d, s, bands), f"{name} {part[0]}")


# ---- alpha quantisation at every edge -------------------------------------------------------------------------------------
EDGE_SETS = {255: None, 1023: None, 4095: None,
             65535: sorted(set(range(0, 300)) | set(range(65235, 65536)) | set(range(0, 65536, 97)))}


def rgb_edge_frames(fmt, n):
    """one row per pad alpha: source alpha byte 255 (so that SOURCE writes the integer pad alpha itself) and every colour
    pair in the other bytes; destination alpha varied"""
    ai = cd.RGB[fmt][1]
    ci = [c for c in range(4) if c != ai]
    s_c, d_c = cd.pair_grid(3 * 256)
    s, d = np.zeros((n, 256, 4), np.uint8), np.zeros((n, 256, 4), np.uint8)
    s[:, :, ci] = s_c.reshape(256, 3)
    d[:, :, ci] = d_c.reshape(256, 3)
    s[:, :, ai] = 255
    s[:, ::2, ai] = np.arange(128, dtype=np.uint8) * 2
    d[:, :, ai] = np.arange(256, dtype=np.uint8)[::-1]
    return d, s


def yuv_edge_frames(nbits, n):
    """one row per pad alpha of [3, n, 256] samples: the extremes of the range against each other and structured pairs"""
    r = (1 << nbits) - 1
    v = np.array(structured(nbits, 28), np.int64)
    sv, dv = np.meshgrid(v, v)
    sv, dv = np.concatenate([[r, 0, r, 0], sv.ravel()])[: 3 * 256], np.concatenate([[0, r, r, 0], dv.ravel()])[: 3 * 256]
    dt = np.uint8 if nbits == 8 else np.int32
    s = np.broadcast_to(np.resize(sv, 3 * 256).reshape(3, 1, 256), (3, n, 256)).astype(dt)
    d = np.broadcast_to(np.resize(dv, 3 * 256).reshape(3, 1, 256), (3, n, 256)).astype(dt)
    return d, s


def edge_calls_rgb(alphas, fmt):
    """(d, s, bands, bg) per call: SOURCE, OVER (opaque) and OVER / ADD (transparent) rows at every edge alpha; alphas
    above 1.0 for OVER"""
    calls = []
    ops = [(cd.SOURCE, cd.WHITE), (cd.OVER, cd.CHECKER), (cd.ADD, cd.TRANSPARENT)]
    for op, bg in ops:
        al = alphas + ([1.0 + 1e-9, 1.5, 3.0] if op == cd.OVER else [])
        for part in cd.chunks(al, cd.MAX_PADS - 1):
            d, s = rgb_edge_frames(fmt, len(part))
            calls.append((d, s, cd.bands_of(part, 1, op), bg))
    return calls


def edge_calls_yuv(rng, nbits, ks=None):
    """(d, s, bands) per call: every edge of `ks` (EDGE_SETS[rng] when None) and alphas above 1.0"""
    ks = EDGE_SETS[rng] if ks is None else ks
    alphas = cd.alpha_edges(rng, ks) + [1.0 + 1e-9, 2.0]
    calls = []
    for part in cd.chunks(alphas, cd.MAX_PADS - 1):
        d, s = yuv_edge_frames(nbits, len(part))
        calls.append((d, s, cd.bands_of(part, 1, cd.OVER)))
    return calls


EDGE_YUV = [(255, "Y444"), (1023, "Y444_10LE"), (4095, "Y444_12LE"), (65535, "Y444_16LE")]


def test_alpha_edges_oracle():
    """the model's quantisation (int (alpha * range), clamped; 1.0 copies) is the oracle's at every edge"""
    for fmt in ("BGRA", "ARGB"):
        for d, s, bands, bg in edge_calls_rgb(cd.alpha_edges(255), fmt):
            check(checker_rgb("oracle", fmt, bg, d, s, bands), cd.rgb_expected(fmt, bg, d, s, bands), f"{fmt} {bands[0]}")
    for rng, name in EDGE_YUV:
        for d, s, bands in edge_calls_yuv(rng, cd.YUV[name][1]):
            check(checker_yuv("oracle", name, d, s, bands), cd.yuv_expected(cd.YUV[name][1], d, s, bands), f"{name} {bands[0]}")


@pytest.mark.ref
def test_alpha_edges_ref():
    for d, s, bands, bg in edge_calls_rgb(cd.alpha_edges(255), "BGRA"):
        check(checker_rgb("ref", "BGRA", bg, d, s, bands), checker_rgb("oracle", "BGRA", bg, d, s, bands), f"{bands[0]}")
    for rng, name in EDGE_YUV:
        calls = edge_calls_yuv(rng, cd.YUV[name][1])
        for d, s, bands in calls[:: max(1, len(calls) // 20)]:
            check(checker_yuv("ref", name, d, s, bands), checker_yuv("oracle", name, d, s, bands), f"{name} {bands[0]}")


# ---- the emulated kernels ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    import build_emu
    from gstreamer_b200 import _lib
    lib = C.CDLL(build_emu.build())
    for name, (res, args) in _lib._SIGS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return cd.Host(lib)


# the emulator runs a call in about half a second: every edge at 255, sampled edges at the wider ranges (the GPU file runs
# every one; the quantisation is host code both builds share)
EMU_EDGES = {255: None, 1023: list(range(0, 1024, 31)) + [1022, 1023], 4095: list(range(0, 4096, 127)) + [4094, 4095],
             65535: [0, 1, 2, 32767, 32768, 65534, 65535]}


@pytest.mark.parametrize("entry", ["blend", "convert"])
def test_alpha_edges_emulated(emu, entry):
    """edge alphas through b200_comp_blend / b200_comp_blend_yuv (entry "blend") and b200_comp_blend_convert"""
    calls = edge_calls_rgb(cd.alpha_edges(255), "BGRA")
    for d, s, bands, bg in [c for c in calls if c[2][0][3] == cd.SOURCE] + [c for c in calls if c[2][-1][2] > 1.0]:
        check(cd.rgb_pads(emu, "BGRA", bg, d, s, bands, entry=entry), cd.rgb_expected("BGRA", bg, d, s, bands), f"{bands[0]}")
    for rng, name in EDGE_YUV:
        for d, s, bands in edge_calls_yuv(rng, cd.YUV[name][1], EMU_EDGES[rng]):
            got = cd.yuv_pads(emu, name, d, s, bands, "yuv" if entry == "blend" else "convert")
            check(got, cd.yuv_expected(cd.YUV[name][1], d, s, bands), f"{name} {bands[0]}")


@pytest.mark.parametrize("fmt", ["RGBA", "ARGB"])
def test_emulated_rgb(emu, fmt):
    """comp_kernel's BLEND, SOURCE, OVERLAY and OVERLAY_ADD on reduced domains: all (s, d) at a few source alphas, the
    (as, dalpha) grid, and every (as, dalpha) under a spread of pad alphas"""
    d, s = blend_domain(fmt, (0, 1, 128, 254, 255))
    for bg, op in ((cd.BLACK, cd.OVER), (cd.TRANSPARENT, cd.OVER), (cd.TRANSPARENT, cd.ADD)):
        bands = [(0, d.shape[0], 1.0, op)]
        check(cd.rgb_pads(emu, fmt, bg, d, s, bands), cd.rgb_expected(fmt, bg, d, s, bands), f"{bg} {op}")
    ks = list(range(1, 256, 4)) + [255]
    for op, bg in ((cd.SOURCE, cd.WHITE), (cd.OVER, cd.BLACK), (cd.OVER, cd.TRANSPARENT), (cd.ADD, cd.TRANSPARENT)):
        for part in cd.chunks(ks, cd.MAX_PADS - 1):
            d, s = alpha_domain(fmt, part, rows=4)
            bands = cd.bands_of([cd.alpha_for(k, 255) for k in part], 4, op)
            check(cd.rgb_pads(emu, fmt, bg, d, s, bands), cd.rgb_expected(fmt, bg, d, s, bands), f"{op} {bg}")


@pytest.mark.parametrize("name", list(cd.YUV))
def test_emulated_planes(emu, name):
    """comp_yuv_kernel: all 8-bit (s, d) at a spread of alphas; wide blends on structured in-range and out-of-range pairs"""
    nbits = cd.YUV[name][1]
    r = (1 << nbits) - 1
    if nbits == 8:
        ks, values = list(range(1, 256, 16)) + [255], None
    else:
        ks, values = wide_alphas(nbits, 8, seed=3), structured(nbits, 256, full=True)
    d, s, rows = plane_domain(nbits, 1 << 16, len(ks), values)
    bands = cd.bands_of([cd.alpha_for(k, r) for k in ks], rows, cd.OVER)
    check(cd.yuv_pads(emu, name, d, s, bands), cd.yuv_expected(nbits, d, s, bands), name)


# ---- launch chunks and the pad limit (run here on the emulated library, and by tests/test_comp_domain_gpu.py) -------------
# b200_comp_blend launches every 32 pads and b200_comp_blend_yuv every 24; each later launch continues from the destination,
# through a scalar path for rows that are not 16-byte aligned, W % 4 != 0 and the last n < 4 pixels of a row
RGB_CHUNK = [(n, W) for n in (31, 32, 33, 63, 64) for W in (129, 130, 131)]
YUV_CHUNK = [(n, name) for n in (23, 24, 25, 48, 49, 64) for name in ("Y444", "Y444_16LE")]


def untouched(buf, offset, rows, row_bytes, stride, fill=0x5A):
    """every byte of the allocation outside the frame's rows still holds `fill`"""
    keep = np.ones(buf.size, bool)
    keep[offset: offset + rows * stride].reshape(rows, stride)[:, :row_bytes] = False
    return bool((buf[keep] == fill).all())


def run_rgb_chunk(mem, n, W, entry="blend"):
    """n pads (pad 0 copying the destination, n - 1 random ones) into a W-wide destination that starts 4 bytes into its
    allocation, at a row stride of 4 modulo 16"""
    rng = np.random.default_rng(1000 * n + W)
    H, fmt, bg = 21, ("BGRA", "ARGB")[n % 2], (cd.BLACK, cd.TRANSPARENT, cd.CHECKER)[W % 3]
    row_pad = (4 - 4 * W) % 16 or 16
    assert (4 * W + row_pad) % 16 == 4
    d = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    pads = cd.random_pads(rng, W, H, n - 1)
    st, buf, got = cd.rgb_pads_call(mem, fmt, bg, d, pads, entry, dst_offset=4, row_pad=row_pad)
    assert st == 0, st
    check(got, cd.rgb_expected_pads(fmt, bg, d, pads), f"{entry} {n} pads W {W}")
    assert untouched(buf, 4, H, 4 * W, 4 * W + row_pad)


def run_yuv_chunk(mem, n, name, entry="yuv"):
    nbits = cd.YUV[name][1]
    rng = np.random.default_rng(n + nbits)
    W, H = 37, 19
    d = rng.integers(0, 1 << nbits, (3, H, W)).astype(np.uint8 if nbits == 8 else np.int32)
    pads = cd.random_pads(rng, W, H, n - 1, planes=3, nbits=nbits)
    st, buf, got = cd.yuv_pads_call(mem, name, d, pads, entry)
    assert st == 0, st
    check(got, cd.yuv_expected_pads(nbits, d, pads), f"{entry} {name} {n} pads")
    es = 1 if nbits == 8 else 2
    assert untouched(buf, 0, 3 * H, W * es, W * es + 4)


def run_too_many_pads(mem):
    """65 pads: every entry point refuses the call and leaves the destination byte for byte as it was"""
    rng = np.random.default_rng(65)
    d = rng.integers(0, 256, (9, 13, 4), dtype=np.uint8)
    pads = cd.random_pads(rng, 13, 9, 64)
    for entry in ("blend", "convert"):
        st, buf, _ = cd.rgb_pads_call(mem, "BGRA", cd.BLACK, d, pads, entry)
        assert st < 0 and (buf == 0x5A).all(), (entry, st)
    d = rng.integers(0, 256, (3, 9, 13)).astype(np.uint8)
    pads = cd.random_pads(rng, 13, 9, 64, planes=3)
    for entry in ("yuv", "convert"):
        st, buf, _ = cd.yuv_pads_call(mem, "Y444", d, pads, entry)
        assert st < 0 and (buf == 0x5A).all(), (entry, st)


@pytest.mark.parametrize("n,W", RGB_CHUNK)
def test_rgb_chunks_emulated(emu, n, W):
    run_rgb_chunk(emu, n, W, "blend" if n % 2 else "convert")


@pytest.mark.parametrize("n,name", YUV_CHUNK)
def test_yuv_chunks_emulated(emu, n, name):
    run_yuv_chunk(emu, n, name, "yuv" if n % 2 else "convert")


def test_too_many_pads_emulated(emu):
    run_too_many_pads(emu)
