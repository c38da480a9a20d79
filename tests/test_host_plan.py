"""Host-side plan builders of the product (C++, no device needed: device=-1) against the oracle:
tap tables, stage order, matrix, chroma pairing, specialised-kernel eligibility, audio filter."""
import ctypes as C

import numpy as np
import pytest

from oracle import bindings as ob

SIZES = [(3840, 2160, 1920, 1080), (1920, 1080, 1280, 720), (641, 481, 111, 30), (111, 30, 641, 481),
         (100, 100, 150, 50), (640, 480, 320, 240), (17, 33, 64, 7), (64, 48, 64, 48), (40, 90, 40, 31)]


def _oracle_taps(method, insz, outsz, prec):
    o = ob.oracle()
    m, mt, bc = ob.ELEMENT_METHODS[method]
    rs = ob.RS(m, mt, 0, 2.0, 1.0, 0.0, 1 / 3, 1 / 3)
    if bc:
        rs.cubic_b, rs.cubic_c = bc
    off = np.zeros(outsz, dtype=np.uint32)
    t = np.zeros(outsz * 128)
    n = o.oracle_resampler_taps(C.byref(rs), insz, outsz, off.ctypes.data, t.ctypes.data)
    t = t[: outsz * n].reshape(outsz, n)
    q = np.zeros((outsz, n), dtype=np.int16)
    for i in range(outsz):
        row = np.ascontiguousarray(t[i])
        qq = np.zeros(n, dtype=np.int16)
        o.oracle_quantize_taps(row.ctypes.data, qq.ctypes.data, n, prec)
        q[i] = qq
    return n, off, q


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d-%dx%d" % s)
@pytest.mark.parametrize("method", range(10))
def test_tap_tables_and_order(size, method):
    import gstreamer_b200 as g
    iw, ih, ow, oh = size
    el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=-1)
    el.set_info(g.VideoInfo(23, iw, ih), g.VideoInfo(12, ow, oh))
    pi = el.plan_info()
    for d, (a, b) in enumerate([(iw, ow), (ih, oh)]):
        off, coef = el.taps(d)
        if a == b:
            assert (off == np.arange(b)).all()
            continue
        n, ooff, oq = _oracle_taps(method, a, b, 6)
        assert (pi.h_taps, pi.v_taps)[d] == n
        if n >= 3:
            assert (off == ooff).all() and (coef == oq).all()
        elif n == 1:
            assert (off == ooff).all()
        elif d == 1:                      # vertical 2-tap: centre aligned, 8-bit second tap
            n, ooff, oq = _oracle_taps(method, a, b, 8)
            assert (off == ooff).all() and (coef[:, 0] == oq[:, 1]).all()
        else:                             # horizontal 2-tap: edge aligned 16.16 stepping
            inc = 0 if b == 1 else ((a - 1) << 16) // (b - 1) - 1
            x = np.arange(b, dtype=np.int64) * inc
            assert (off == (x >> 16)).all() and (coef[:, 0] == ((x >> 8) & 0xff)).all()
    # chain_scale ordering (video-converter.c:1685-1718)
    assert pi.matrix_first == int(ow * oh > iw * ih)
    assert pi.h_first == int(ow * ih <= iw * oh)
    d = ob.vcs_desc(iw, ih, ow, oh, method)
    p = (C.c_int * 5)()
    im = (C.c_int * 16)()
    assert ob.oracle().oracle_vcs_matrix(C.byref(d), p, im) == 0
    assert list(pi.p) == list(p)


@pytest.mark.parametrize("matrix,rng", [(2, 1), (2, 2), (3, 1), (3, 2), (4, 1), (4, 2), (5, 2), (6, 1), (6, 2)])
def test_matrix_all_colorimetries(matrix, rng):
    import gstreamer_b200 as g
    el = g.CudaVideoConvertScale(add_borders=False, method=3, cuda_device_id=-1)
    el.set_info(g.VideoInfo(23, 64, 48).set_colorimetry(matrix=matrix, range=rng), g.VideoInfo(12, 32, 24))
    d = ob.vcs_desc(64, 48, 32, 24, 3, matrix=matrix, rng=rng)
    p = (C.c_int * 5)()
    im = (C.c_int * 16)()
    assert ob.oracle().oracle_vcs_matrix(C.byref(d), p, im) == 0
    assert list(el.plan_info().p) == list(p)


def test_chroma_plan_standard_and_skipping():
    import gstreamer_b200 as g
    el = g.CudaVideoConvertScale(add_borders=False, method=3, cuda_device_id=-1)
    el.set_info(g.VideoInfo(23, 64, 48), g.VideoInfo(12, 32, 24))
    m = el.chroma_plan()
    assert m[0] == 0 and (m[1::2] == 1).all() and (m[2::2] == 2).all()
    # nearest 2:1 skips lines: a requested even line opens its own pair (SURVEY appendix A-4)
    el = g.CudaVideoConvertScale(add_borders=False, method=0, cuda_device_id=-1)
    el.set_info(g.VideoInfo(23, 640, 480), g.VideoInfo(12, 320, 240))
    off, _ = el.taps(1)
    m = el.chroma_plan()
    assert off[122] == 244 and off[123] == 246          # the floating point floor lands on even lines here
    assert m[244] == 2 and m[246] == 1 and m[245] == 0 and m[1] == 1


def test_specialised_kernel_eligibility():
    import gstreamer_b200 as g

    def eligible(iw, ih, ow, oh, method, site=2, **kw):
        el = g.CudaVideoConvertScale(add_borders=False, method=method, cuda_device_id=-1)
        ii = g.VideoInfo(23, iw, ih).set_colorimetry(chroma_site=site)
        if "stride" in kw:
            ii.set_layout([kw["stride"], kw["stride"]], [0, kw["stride"] * ih])
        el.set_info(ii, g.VideoInfo(12, ow, oh))
        try:
            el.set_kernel_variant(1)
            return True
        except g.B200Error:
            return False

    assert eligible(3840, 2160, 1920, 1080, 3)
    assert eligible(1920, 1080, 960, 540, 9)
    assert not eligible(3840, 2160, 1920, 1080, 1)            # bilinear: 2 taps
    assert not eligible(3840, 2160, 1280, 720, 3)             # 3:1
    assert not eligible(3840, 2160, 1920, 1080, 3, site=1)    # not h-cosited
    assert not eligible(644, 480, 322, 240, 3)                # width not a multiple of 8
    assert not eligible(640, 480, 320, 240, 3, stride=644)    # rows not 8-byte aligned
    assert not eligible(640, 480, 320, 240, 0)                # nearest


@pytest.mark.parametrize("cfg", [(48000, 44100, 4), (44100, 48000, 4), (8000, 16000, 0), (22050, 48000, 9),
                                 (96000, 8000, 7), (48000, 24000, 10), (101, 99, 4)])
def test_audio_filter_design(cfg):
    from gstreamer_b200.audio import CudaAudioResample
    a, b, q = cfg
    o = ob.oracle()
    rs = CudaAudioResample(quality=q, cuda_device_id=-1)
    rs.set_caps(a, b, 2)
    pi = rs.plan_info()
    ho = o.oracle_ars_new(a, b, 2, q)
    v = [C.c_int() for _ in range(6)]
    o.oracle_ars_info(ho, *[C.byref(x) for x in v])
    assert [pi.n_taps, pi.n_phases, pi.in_step, pi.out_step, pi.filter_mode, pi.oversample] == [x.value for x in v]
    for ph in range(pi.n_phases):
        t = np.zeros(pi.n_taps, dtype=np.float32)
        o.oracle_ars_phase_taps(ho, ph, t.ctypes.data)
        assert np.array_equal(t.view(np.uint32), rs.phase_taps(ph).view(np.uint32)), f"phase {ph}"
    # framing arithmetic before any data: get_out_frames for a few sizes
    for n in (1, 100, 480, 4800):
        assert rs.get_out_frames(n) == o.oracle_ars_get_out_frames(ho, n)
        assert rs.get_in_frames(n) == o.oracle_ars_get_in_frames(ho, n)
    assert rs.max_latency == o.oracle_ars_max_latency(ho)
    o.oracle_ars_free(ho)


def test_c5_filter_numbers_from_the_survey():
    """SURVEY §8a-14: 48k -> 44.1k at quality 4: steps 160/147, 72 taps, 147 phases, FULL mode"""
    from gstreamer_b200.audio import CudaAudioResample
    rs = CudaAudioResample(quality=4, cuda_device_id=-1)
    rs.set_caps(48000, 44100, 256)
    pi = rs.plan_info()
    assert (pi.in_step, pi.out_step, pi.n_taps, pi.n_phases, pi.filter_mode, pi.oversample) == (160, 147, 72, 147, 1, 8)


def test_fast_kernel_selection_sweep():
    """host-only plans over random sizes, methods and input formats: the fast kernels' shape searches
    (light_geometry, search_tile_shape) check every output's window against its tile's staged range and take
    no shape that leaves it, which would fall back to the generic kernel — for default layouts that must
    never happen for the common methods at moderate ratios, and every plan must build"""
    import gstreamer_b200 as g
    rng = np.random.default_rng(0)
    counts = {}
    for t in range(1500):
        iw, ih = int(rng.integers(1, 2000)), int(rng.integers(1, 1200))
        uniform = rng.random() < 0.6
        if uniform:
            f = rng.uniform(0.25, 4.0)
            ow, oh = max(1, int(iw * f)), max(1, int(ih * f))
        else:
            ow, oh = int(rng.integers(1, 2000)), int(rng.integers(1, 1200))
        m = int(rng.integers(0, 10))
        fmt = int(rng.choice([23, 24, 2, 3]))
        el = g.CudaVideoConvertScale(add_borders=False, method=m, cuda_device_id=-1)
        el.set_info(g.VideoInfo(fmt, iw, ih), g.VideoInfo(12, ow, oh))
        v = int(el.plan_info().kernel_variant)
        counts[v] = counts.get(v, 0) + 1
        if m in (0, 1):
            assert v == 2, (iw, ih, ow, oh, m, fmt)          # nearest / bilinear: light kernel, either order
        elif uniform and m in (3, 9) and min(iw, ih) >= 16:
            assert v in (1, 3), (iw, ih, ow, oh, m, fmt)     # lanczos / mitchell at moderate ratios
        if v == 1:
            assert fmt in (23, 24) and iw == 2 * ow and ih == 2 * oh
    assert counts.get(0, 0) < 0.08 * 1500                    # mixed 2-tap / n-tap axes and extreme ratios only


def test_cross_family_420_plan():
    """NV12 <-> I420 etc.: the chain + chroma down-sampling plan (kernel_variant 5, two launches) builds for every
    method and both pass orders; a differing colour matrix (a matrix stage) is refused"""
    import gstreamer_b200 as g

    def build(fi, fo, iw, ih, ow, oh, m=1, matrix=None, site=None, out_site=None):
        el = g.CudaVideoConvertScale(add_borders=False, method=m, cuda_device_id=-1)
        ii, oi = g.VideoInfo(fi, iw, ih), g.VideoInfo(fo, ow, oh)
        if site is not None:
            ii.set_colorimetry(chroma_site=site)
        oi.set_colorimetry(matrix=ii.c.color_matrix if matrix is None else matrix,
                           chroma_site=ii.c.chroma_site if out_site is None else out_site)
        el.set_info(ii, oi)
        return el.plan_info()

    for fi, fo in [(23, 2), (2, 23), (23, 24), (24, 3), (3, 24)]:
        for size in [(64, 48, 32, 24), (64, 48, 96, 72), (1920, 1080, 1280, 720), (100, 100, 150, 50), (33, 17, 33, 17)]:
            for m in range(10):
                pi = build(fi, fo, *size, m=m)
                assert (int(pi.kernel_variant), int(pi.matrix_first)) == (5, 0)
                assert int(pi.n_launches_per_convert) == 2
                assert int(pi.h_first) == int(size[2] * size[1] <= size[0] * size[3])
    with pytest.raises(g.B200Error):
        build(23, 2, 64, 48, 32, 24, matrix=3)                 # 64x48 defaults to bt601: a matrix stage would be needed
    # odd height and no vertical scaler: a third launch rebuilds the line the down-sampler's last pair reads past the
    # frame - unless the input chroma is vertically co-sited (nothing to rebuild) or no resampler exists at all
    assert int(build(23, 2, 64, 49, 32, 49).n_launches_per_convert) == 3
    assert int(build(23, 2, 64, 49, 32, 49, site=4, out_site=4).n_launches_per_convert) == 2
    assert int(build(23, 2, 64, 49, 64, 49).n_launches_per_convert) == 2
    assert int(build(23, 2, 64, 49, 64, 49, out_site=2).n_launches_per_convert) == 3
    # the same-family pairs keep their plane-scaling plan
    assert int(build(23, 23, 64, 48, 32, 24).kernel_variant) == 4


def test_transfer_colorimetry_from_input():
    """1080p (bt709, mpeg2 site) -> 480p I420: the caps defaults of the small size would be bt601 / site none; the
    element's fixation carries the input's over, which is what makes the chain matrix-free"""
    import gstreamer_b200 as g
    ii, oi = g.VideoInfo(23, 1920, 1080), g.VideoInfo(2, 854, 480)
    assert (oi.c.color_matrix, oi.c.chroma_site) == (4, 1)
    el = g.CudaVideoConvertScale(add_borders=False, method=1, cuda_device_id=-1)
    with pytest.raises(g.B200Error):
        el.set_info(ii, oi)
    g.transfer_colorimetry_from_input(ii, oi)
    assert (oi.c.color_matrix, oi.c.color_range, oi.c.chroma_site) == (3, 2, 2)
    el.set_info(ii, oi)
    assert int(el.plan_info().kernel_variant) == 5
    rgb = g.VideoInfo(12, 854, 480)
    g.transfer_colorimetry_from_input(ii, rgb)
    assert rgb.c.color_matrix == 1


def test_rgb_input_plan_matches_the_oracle_matrix(monkeypatch):
    """packed RGB -> 4:2:0 (generic kernel + chroma down-sampling; device-verified in tests/test_vcs_rgbin_gpu.py):
    the host plan carries the same x256 RGB -> YUV matrix as the oracle for
    every output colorimetry, sits the matrix between the shrinking and the growing scalers, and never needs the
    odd-height third launch"""
    import gstreamer_b200 as g

    def build(fi, fo, iw, ih, ow, oh, m=1, **out_colorimetry):
        el = g.CudaVideoConvertScale(add_borders=False, method=m, cuda_device_id=-1)
        ii, oi = g.VideoInfo(fi, iw, ih), g.VideoInfo(fo, ow, oh)
        if out_colorimetry:
            oi.set_colorimetry(**out_colorimetry)
        el.set_info(ii, oi)
        return el

    im = (C.c_int * 16)()
    for fi in (7, 8, 9, 10, 11, 12, 13, 14):
        for fo in (2, 3, 23, 24):
            for size in [(64, 48, 32, 24), (64, 48, 96, 72), (1920, 1080, 1280, 720), (33, 17, 33, 17), (64, 49, 32, 49)]:
                el = build(fi, fo, *size)
                pi = el.plan_info()
                assert (int(pi.kernel_variant), int(pi.n_launches_per_convert)) == (5, 2)
                assert int(pi.matrix_first) == int(size[2] * size[3] > size[0] * size[1])
                d = ob.vcs_desc(*size, 1, in_fmt=fi, out_fmt=fo)
                assert ob.oracle().oracle_vcs_matrix_rgb2yuv(C.byref(d), im) == 0
                assert el.matrix().ravel().tolist() == list(im)
    for matrix in (2, 3, 4, 5, 6):
        for rng in (1, 2):
            el = build(12, 23, 64, 48, 32, 24, matrix=matrix, range=rng, chroma_site=6)
            d = ob.vcs_desc(64, 48, 32, 24, 1, in_fmt=12, out_fmt=23)
            d.out_matrix, d.out_range = matrix, rng
            assert ob.oracle().oracle_vcs_matrix_rgb2yuv(C.byref(d), im) == 0
            assert el.matrix().ravel().tolist() == list(im)
    # the same format at another size (a compositor's scaled pads): the one-plane scaling rows; another byte order: the
    # matrix-free chain, same kernel with a byte swizzle and the chain's pass-order rule
    for m in range(10):
        for size in [(64, 48, 32, 24), (40, 30, 64, 48), (100, 100, 150, 50), (64, 48, 64, 48)]:
            assert int(build(11, 11, *size, m=m).plan_info().kernel_variant) == 4
            assert int(build(12, 11, *size, m=m).plan_info().kernel_variant) == 4


def test_add_borders_rectangle_and_plan():
    """the mirror's add-borders geometry equals the oracle's (both restate gstvideoconvertscale.c:920-952), the plan then
    describes the rectangle (tap tables of the rectangle's size) and one more launch for the border fill"""
    import gstreamer_b200 as g
    rng = np.random.default_rng(3)
    for t in range(200):
        iw, ih, ow, oh = (int(v) for v in rng.integers(2, 400, 4))
        el = g.CudaVideoConvertScale(method=3, cuda_device_id=-1, add_borders=True)
        x, y, w, h = ob.vcs_borders(iw, ih, ow, oh)
        if w < 1 or h < 1:
            continue
        el.set_info(g.VideoInfo(23, iw, ih), g.VideoInfo(12, ow, oh))
        assert (el.borders_w // 2, el.borders_h // 2, ow - el.borders_w, oh - el.borders_h) == (x, y, w, h)
        pi = el.plan_info()
        bordered = (w, h) != (ow, oh)
        assert int(pi.n_launches_per_convert) == (2 if bordered else 1)
        n, off, q = _oracle_taps(3, iw, w, 6) if iw != w else (0, None, None)
        assert int(pi.h_taps) == n
    # explicit rectangle through the C-ABI config; 4:2:0 outputs round the origin down to even
    from gstreamer_b200 import _lib
    cfg = _lib.VcsConfigC()
    g.lib.b200_vcs_config_init(C.byref(cfg))
    assert (cfg.border_argb, cfg.fill_border) == (0xff000000, 1)
    cfg.dest_x, cfg.dest_y, cfg.dest_width, cfg.dest_height = 5, 3, 20, 10
    h = C.c_void_p()
    ii, oi = g.VideoInfo(23, 64, 48), g.VideoInfo(23, 40, 30)
    assert g.lib.b200_vcs_create(C.byref(ii.c), C.byref(oi.c), C.byref(cfg), -1, C.byref(h)) == 0
    g.lib.b200_vcs_destroy(h)
    cfg.dest_x = 39                                            # clipped to the frame: 1 column left
    assert g.lib.b200_vcs_create(C.byref(ii.c), C.byref(oi.c), C.byref(cfg), -1, C.byref(h)) == 0
    g.lib.b200_vcs_destroy(h)
    cfg.dest_x = 41                                            # rounds down to 40 = outside: empty rectangle
    assert g.lib.b200_vcs_create(C.byref(ii.c), C.byref(oi.c), C.byref(cfg), -1, C.byref(h)) == -1


def test_remaining_element_properties_are_accepted_at_their_defaults():
    import gstreamer_b200 as g
    ii, oi = g.VideoInfo(23, 64, 48), g.VideoInfo(12, 32, 24)
    g.CudaVideoConvertScale(add_borders=False, cuda_device_id=-1, n_threads=8, dither="none", chroma_resampler="linear", alpha_value=1.0).set_info(ii, oi)
    for kw in ({"chroma_resampler": "cubic"}, {"alpha_mode": "set"}, {"alpha_value": 0.5}, {"gamma_mode": "remap"},
               {"primaries_mode": "fast"}, {"matrix_mode": "none"}, {"chroma_mode": "none"}, {"dither_quantization": 4}):
        with pytest.raises(g.B200Error) as e:
            g.CudaVideoConvertScale(add_borders=False, cuda_device_id=-1, **kw).set_info(ii, oi)
        assert e.value.status == -2
    with pytest.raises(TypeError):
        g.CudaVideoConvertScale(add_borders=False, no_such_property=1)


def test_compositor_pad_sizing_policy():
    """_mixer_pad_get_output_size (compositor.c:289-417) at pixel aspect ratio 1/1"""
    from gstreamer_b200.compositor import pad_output_size, CudaCompositorPad
    import gstreamer_b200 as g
    assert pad_output_size(1920, 1080, 0, 0) == (1920, 1080, 0, 0)                       # unset: unscaled
    assert pad_output_size(1920, 1080, 640, 640) == (640, 640, 0, 0)                     # policy none: stretched
    assert pad_output_size(1920, 1080, 640, 640, "keep-aspect-ratio") == (640, 360, 0, 140)
    assert pad_output_size(640, 480, 1920, 1080, "keep-aspect-ratio") == (1440, 1080, 240, 0)
    assert pad_output_size(1920, 1080, 1280, 720, "keep-aspect-ratio") == (1280, 720, 0, 0)
    assert pad_output_size(1000, 3, 10, 100, "keep-aspect-ratio") == (0, 0, 0, 0)        # rounds to an empty picture
    assert pad_output_size(100, 100, 0, 50, zero_size_is_unscaled=False) == (0, 0, 0, 0)
    pad = CudaCompositorPad(640, 640, xpos=10, ypos=20, in_info=g.VideoInfo(23, 1920, 1080), sizing_policy="keep-aspect-ratio")
    assert (pad.width, pad.height, pad.x_offset, pad.y_offset, pad.stride) == (640, 360, 0, 140, 2560)


def test_audioresample_remaining_properties(monkeypatch):
    import gstreamer_b200 as g
    from gstreamer_b200.audio import CudaAudioResample
    CudaAudioResample(cuda_device_id=-1, resample_method="kaiser", sinc_filter_auto_threshold=1).set_caps(48000, 44100, 2)
    # equal rates: pass-through like the element (no resampler behind it); the library itself follows gst_audio_resampler
    # (every output = the first sample of its window) in opt-in device code
    rs = CudaAudioResample(cuda_device_id=-1)
    rs.set_caps(44100, 44100, 2)
    assert rs.passthrough
    with pytest.raises(g.B200Error):
        rs.transform(None, 10, None, 10)
    from gstreamer_b200 import _lib
    cfg, h = _lib.ArsConfigC(), C.c_void_p()
    cfg.in_rate, cfg.out_rate, cfg.channels, cfg.quality = 48000, 48000, 2, 4
    assert g.lib.b200_ars_create(C.byref(cfg), -1, C.byref(h)) == 0     # the library follows gst_audio_resampler (copy kernel)
    g.lib.b200_ars_destroy(h)
    # every method / table interpolation / filter mode builds a plan (device-verified in tests/test_ars_options_gpu.py)
    CudaAudioResample(cuda_device_id=-1, sinc_filter_interpolation="linear").set_caps(48000, 44100, 2)
    for kw in ({"resample_method": "linear"}, {"resample_method": "nearest"}, {"resample_method": "cubic"},
               {"sinc_filter_interpolation": "linear", "sinc_filter_mode": "interpolated"}):
        CudaAudioResample(cuda_device_id=-1, **kw).set_caps(48000, 44100, 2)


@pytest.mark.parametrize("method,mode,interp", [("blackman-nuttall", "auto", "cubic"), ("blackman-nuttall", "full", "none"),
                                                ("kaiser", "full", "cubic"), ("kaiser", "full", "none"),
                                                ("kaiser", "interpolated", "cubic"), ("kaiser", "interpolated", "none"),
                                                ("blackman-nuttall", "interpolated", "cubic"), ("kaiser", "auto", "none"),
                                                ("kaiser", "full", "linear"), ("blackman-nuttall", "auto", "linear"),
                                                ("kaiser", "interpolated", "linear"),
                                                ("nearest", "auto", "cubic"), ("linear", "auto", "cubic"),
                                                ("cubic", "interpolated", "linear")])
def test_audio_method_and_filter_mode_plans(method, mode, interp, monkeypatch):
    """host plan == oracle (pinned to the reference for these options) for the filter design, the mode decision and -
    FULL mode, F32 - every phase's taps bit for bit"""
    from gstreamer_b200.audio import CudaAudioResample
    o = ob.oracle()
    M = {"nearest": 0, "linear": 1, "cubic": 2, "blackman-nuttall": 3, "kaiser": 4}
    MO = {"interpolated": 0, "full": 1, "auto": 2}
    I = {"none": 0, "linear": 1, "cubic": 2}
    for (a, b, q) in [(48000, 44100, 4), (44100, 48000, 6), (8000, 16000, 0), (96000, 44100, 8), (101, 99, 10), (3, 2, 5),
                      (48000, 8000, 1)]:
        rs = CudaAudioResample(quality=q, cuda_device_id=-1, resample_method=method, sinc_filter_mode=mode,
                               sinc_filter_interpolation=interp)
        rs.set_caps(a, b, 2)
        pi = rs.plan_info()
        ho = o.oracle_ars_new_opts(a, b, 2, q, 0, M[method], MO[mode], I[interp])
        v = [C.c_int() for _ in range(6)]
        o.oracle_ars_info(ho, *[C.byref(x) for x in v])
        assert [pi.n_taps, pi.n_phases, pi.in_step, pi.out_step, pi.filter_mode, pi.oversample] == [x.value for x in v]
        for ph in range(0, pi.n_phases, max(1, pi.n_phases // 50)):
            t = np.zeros(pi.n_taps, dtype=np.float32)
            o.oracle_ars_phase_taps(ho, ph, t.ctypes.data)
            assert np.array_equal(t.view(np.uint32), rs.phase_taps(ph).view(np.uint32)), f"phase {ph}"
        o.oracle_ars_free(ho)


def test_packed_422_to_420_plan():
    """capture -> encoder: YUY2 / UYVY -> I420 / YV12 at an unchanged size is the reference's table row (one launch,
    vcs_yuy2_420_kernel); any other pair or size the chain; a border rectangle disables the table row; the output keeps
    the chroma-site default of its own size (the fixation does not carry it across a sub-sampling change); planar
    4:2:2 / 4:4:4 -> planar 4:2:0 are plane-scaling rows"""
    import gstreamer_b200 as g
    from gstreamer_b200.video import transfer_colorimetry_from_input

    def build(fi, fo, iw, ih, ow, oh, m=1, site=None, **cfg):
        el = g.CudaVideoConvertScale(add_borders=False, method=m, cuda_device_id=-1, **cfg)
        ii, oi = g.VideoInfo(fi, iw, ih), g.VideoInfo(fo, ow, oh)
        if site is not None:
            ii.set_colorimetry(chroma_site=site)
        transfer_colorimetry_from_input(ii, oi)
        el.set_info(ii, oi)
        return el, ii, oi

    YUY2, UYVY, YVYU, Y42B, Y444, I420, YV12, NV12 = 4, 5, 19, 18, 20, 2, 3, 23
    for fi in (YUY2, UYVY):
        for fo in (I420, YV12):
            el, _, _ = build(fi, fo, 640, 480, 640, 480)
            assert el.kernel_name() == "vcs_yuy2_420_kernel" and int(el.plan_info().n_launches_per_convert) == 1
            el, _, _ = build(fi, fo, 33, 17, 33, 17, m=3)
            assert el.kernel_name() == "vcs_yuy2_420_kernel"
    for fi, fo, size in [(YVYU, I420, (640, 480, 640, 480)), (YUY2, NV12, (640, 480, 640, 480)), (YUY2, I420, (640, 480, 320, 240)),
                         (UYVY, YV12, (64, 48, 96, 72))]:
        el, _, _ = build(fi, fo, *size)
        assert el.kernel_name() != "vcs_yuy2_420_kernel" and int(el.plan_info().kernel_variant) == 5
    # sub-sampling changes: matrix / range travel, the site does not (1080p input site 2 -> 480p output default 1)
    _, ii, oi = build(YUY2, I420, 1920, 1080, 854, 480)
    assert (oi.c.color_matrix, oi.c.color_range) == (ii.c.color_matrix, ii.c.color_range) and oi.c.chroma_site == 1
    # planar 4:2:2 / 4:4:4 -> planar 4:2:0: the reference's plane-scaling rows (kernel_variant 4)
    for fi in (Y42B, Y444):
        for fo in (I420, YV12):
            el, _, _ = build(fi, fo, 64, 48, 64, 48)
            assert int(el.plan_info().kernel_variant) == 4
            el, _, _ = build(fi, fo, 64, 48, 40, 30, m=3)
            assert int(el.plan_info().kernel_variant) == 4
        el, _, oi = build(fi, NV12, 64, 48, 64, 48)                # semi-planar outputs: the chain (kernel_variant 5)
        assert int(el.plan_info().kernel_variant) == 5 and oi.c.chroma_site == 1
    build(Y42B, 12, 64, 48, 64, 48)                              # ... and to packed RGB as before
