"""Worst-case content (tests/worstcase.py) on the CPU checkers: first that the content does what it claims (a float64
model of the FIR puts every target beyond the representable range, and the oracle returns the clamped value there),
then the oracle against the reference build on that content for every route family, at production frame sizes, and on
long audio streams."""
import numpy as np
import pytest

import worstcase as wc
from oracle import bindings as ob
from test_oracle_vs_ref import _one_tap_vertical_inplace, _one_tap_vertical_repeat, _vfirst


# ---- the content reaches the extremes (oracle only) ----------------------------------------------------------------------
@pytest.mark.parametrize("size", [(96, 64, 48, 32), (100, 60, 64, 36), (256, 144, 128, 72), (64, 48, 96, 72), (120, 80, 48, 30),
                                  (1920, 1080, 1280, 720)], ids=lambda s: "%dx%d-%dx%d" % s)
@pytest.mark.parametrize("method", [3, 5, 9])
def test_video_targets_are_beyond_range_and_clamped(size, method):
    """I420 -> I420 (the luma plane scaled on its own): the float64 model equals the oracle on every pixel; at every
    target the un-clamped value lies beyond [0, 255] when the target's taps overshoot (a negative tap in either
    direction), and the oracle's byte is the clamped value"""
    iw, ih, ow, oh = size
    qh = wc.taps(method, iw, ow)[2]
    qv = wc.taps(method, ih, oh)[2]
    for seed in range(2):
        f = wc.frame("I420", "I420", size, method, seed)
        got = ob.oracle_vcs_convert(ob.vcs_desc(iw, ih, ow, oh, method, in_fmt=ob.FMT["I420"], out_fmt=ob.FMT["I420"]), f)
        y_in = f[wc.components("I420", iw, ih)[0]["Y"]]
        y_out = got[wc.components("I420", ow, oh)[0]["Y"]]
        ideal, staged, (ti, tj) = wc.plane_model(y_in, method, ow, oh)
        assert np.array_equal(y_out, staged)
        assert len(ti) >= 2 and len(tj) >= 2
        for i in ti:
            for j in tj:
                v = ideal[i, j]
                if (qh[j] < 0).any() or (qv[i] < 0).any():
                    assert v > 255 or v < 0, (i, j, v)
                else:
                    assert v in (0.0, 255.0), (i, j, v)
                assert y_out[i, j] == (255 if v > 127.5 else 0), (i, j, v)


@pytest.mark.parametrize("fmt", ["F32", "S16", "S32", "F64"])
@pytest.mark.parametrize("cfg", [(48000, 44100, 4), (44100, 48000, 4), (96000, 44100, 4), (48000, 44100, 0), (44100, 48001, 4)],
                         ids=lambda c: "%d-%d-q%d" % c)
def test_audio_targets_saturate(fmt, cfg):
    """the oracle's output at every target of a worst-case stream: past full scale and bit-exact unclamped for F32 / F64,
    the format's extreme for S16 / S32 at the level where the weakest target sums to 1.1x full scale (FULL filter mode;
    the interpolated mode's integer accumulators wrap before that, byte for byte like the reference)"""
    a, b, q = cfg
    ofmt, _, dt, _ = ob.AUDIO_FORMATS[fmt]
    x, aims, l1, full = wc.ars_stream(a, b, q, 3000, 2, 1)
    assert l1 > 1.01
    scale = wc.ars_scale(fmt, (a, b, 2, q))
    o = ob.oracle()
    h = o.oracle_ars_new_fmt(a, b, 2, q, ofmt)
    xs = wc.to_format(x, fmt, scale)
    cap = int(3000 * b / a) + 64
    y = np.zeros((cap, 2), dtype=dt)
    n = o.oracle_ars_process_any(h, xs.ctypes.data, 3000, y.ctypes.data, cap)
    o.oracle_ars_free(h)
    if fmt in ("F32", "F64") or full:
        assert wc.check_saturation(y[:n], aims, fmt) >= 10


# ---- the oracle against the reference build ------------------------------------------------------------------------------
def _ref_convert(fi, fo, size, method, frame, nbytes):
    iw, ih, ow, oh = size
    d = ob.vcs_desc(iw, ih, ow, oh, method, in_fmt=ob.FMT[fi], out_fmt=ob.FMT[fo])
    kw = {}
    if fi not in wc.RGB4 and fo not in wc.RGB4:         # the element's caps fixation: colorimetry carried over
        kw = dict(matrix=d.in_matrix, out_matrix=d.in_matrix, site=d.in_chroma_site,
                  out_site=d.in_chroma_site if wc.subsampled(fi) == (2, 2) else (2 if oh > 576 else 1))
        d.out_chroma_site = kw["out_site"]
    got = ob.oracle_vcs_convert(d, frame)
    r = ob.RefVcs(iw, ih, ow, oh, method, in_fmt=ob.FMT[fi], out_fmt=ob.FMT[fo], **kw)
    want = r.convert(frame, np.zeros(max(nbytes, got.size), dtype=np.uint8))[: got.size]
    r.close()
    return got, want


FAMILIES = [("NV12", "BGRA"), ("I420", "RGBA"), ("NV21", "xRGB"),                  # 4:2:0 -> packed RGB
            ("NV12", "NV12"), ("I420", "YV12"), ("NV21", "NV21"),                  # same-family 4:2:0
            ("NV12", "I420"), ("YV12", "NV21"),                                    # cross-family 4:2:0
            ("BGRA", "NV12"), ("RGBA", "I420"), ("xRGB", "NV21"),                  # packed RGB -> 4:2:0
            ("YUY2", "I420"), ("UYVY", "NV12"), ("YVYU", "YV12"),                  # packed 4:2:2 -> 4:2:0
            ("Y42B", "BGRA"), ("Y444", "RGBA"), ("Y42B", "I420"), ("Y444", "NV12"),    # planar 4:2:2 / 4:4:4 inputs
            ("BGRA", "BGRA"), ("RGBA", "ARGB"), ("ABGR", "BGRx")]                  # packed RGB -> packed RGB
WC_SIZES = [(96, 64, 48, 32), (100, 60, 64, 36), (64, 48, 96, 72), (57, 35, 29, 35), (33, 17, 20, 31)]


@pytest.mark.ref
@pytest.mark.parametrize("pair", FAMILIES, ids=lambda p: "%s-%s" % p)
def test_worst_case_matches_reference(pair):
    """every route family on aimed and random XOR-binary frames, all ten methods: the oracle byte for byte equal to the
    reference, except on the reference's two known defect classes (vertical-first chains, a 1-tap vertical pass that
    repeats lines), which tests/test_oracle_vs_ref.py pins by composition"""
    fi, fo = pair
    checked = 0
    for size in WC_SIZES:
        iw, ih, ow, oh = size
        for method in range(10):
            for seed in (method, 100 + method):
                f = wc.frame(fi, fo, size, method, seed) if seed < 100 else wc.random_binary(fi, size, seed)
                got, want = _ref_convert(fi, fo, size, method, f, ow * oh * 4)
                if not np.array_equal(got, want):
                    chain = not (fi in wc.RGB4 and fo in wc.RGB4)
                    assert chain and (_vfirst(iw, ih, ow, oh) or _one_tap_vertical_inplace(ih, oh, method)
                                      or _one_tap_vertical_repeat(iw, ih, ow, oh, method)), (size, method, seed)
                    continue
                checked += 1
    assert checked >= 60


@pytest.mark.ref
@pytest.mark.parametrize("size", [(100, 100, 150, 50), (64, 66, 64, 31), (40, 90, 40, 31)], ids=lambda s: "%dx%d-%dx%d" % s)
@pytest.mark.parametrize("method", [3, 5, 9])
def test_worst_case_vertical_first_two_step(size, method):
    """vertical-first NV12 -> BGRA on worst-case frames, against the two reference runs that cannot alias (NV12 -> AYUV
    at the same size, then AYUV -> BGRA with scaling), as test_oracle_vs_ref.test_vertical_first_two_step"""
    iw, ih, ow, oh = size
    assert _vfirst(iw, ih, ow, oh)
    d = ob.vcs_desc(iw, ih, ow, oh, method)
    for seed in (1, 101):
        frame = wc.frame("NV12", "BGRA", size, method, seed) if seed < 100 else wc.random_binary("NV12", size, seed)
        r1 = ob.RefVcs(iw, ih, iw, ih, method, out_fmt=ob.FMT["AYUV"], matrix=d.in_matrix, rng=d.in_range,
                       site=d.in_chroma_site, out_matrix=d.in_matrix, out_rng=d.in_range, out_site=0)
        ayuv = r1.convert(frame)
        r1.close()
        r2 = ob.RefVcs(iw, ih, ow, oh, method, in_fmt=ob.FMT["AYUV"], matrix=d.in_matrix, rng=d.in_range, site=0)
        want = r2.convert(ayuv)
        r2.close()
        assert np.array_equal(ob.oracle_vcs_convert(d, frame), want)


PRODUCTION = [(3840, 2160, 1920, 1080), (1920, 1080, 3840, 2160), (7680, 4320, 1920, 1080), (3840, 2160, 1280, 720),
              (4096, 2160, 1920, 1080)]


@pytest.mark.ref
@pytest.mark.parametrize("size", PRODUCTION, ids=lambda s: "%dx%d-%dx%d" % s)
@pytest.mark.parametrize("method", [0, 3, 9])
def test_production_shapes_match_reference(size, method):
    """NV12 -> BGRA at the frame sizes users run, a worst-case frame aimed at the taps: the oracle equals the
    single-threaded reference (the device tests compare with the oracle at these sizes)"""
    iw, ih, ow, oh = size
    frame = wc.frame("NV12", "BGRA", size, method, 7)
    r = ob.RefVcs(iw, ih, ow, oh, method)
    want = r.convert(frame)
    r.close()
    assert np.array_equal(ob.oracle_vcs_convert(ob.vcs_desc(iw, ih, ow, oh, method), frame), want)


# (in, out, channels, quality, buffer frames, buffers): one 960 000-frame buffer, 100 to 600 buffers in sequence,
# quality 10, the interpolated filter mode, 256 channels
LONG_STREAMS = [(48000, 44100, 2, 4, 960000, 1), (44100, 48000, 2, 4, 4800, 600), (96000, 44100, 1, 10, 20000, 100),
                (44100, 48001, 2, 4, 9600, 100), (48000, 44100, 256, 4, 4800, 12)]


@pytest.mark.ref
@pytest.mark.parametrize("cfg", LONG_STREAMS, ids=lambda c: "%d-%d-%dch-q%d-%dx%d" % c)
def test_long_stream_matches_reference(cfg):
    """F32 over long streams - 0.88 M to 3.1 M output frames on one or two channels, 53 k frames of 256 channels -
    with full-scale worst-case windows on every channel in alternate buffers and noise in the others: byte-identical
    buffer for buffer"""
    a, b, ch, q, n, count = cfg
    o, r = ob.oracle(), ob.ref()
    ho, hr = o.oracle_ars_new(a, b, ch, q), r.ref_ars_new(a, b, ch, q)
    x, _, _, _ = wc.ars_stream(a, b, q, min(n, 20000), ch, 3)
    rng = np.random.default_rng(a + b + ch)
    total = 0
    try:
        for k in range(count):
            if k == 0 or k % 2:
                buf = np.ascontiguousarray(np.resize(x.astype(np.float32), (n, ch)))
            else:
                buf = ob.audio_test_signal(rng, n, ch, "F32")
            cap = int(n * b / a) + 64
            y1, y2 = np.zeros((cap, ch), dtype=np.float32), np.zeros((cap, ch), dtype=np.float32)
            n1 = o.oracle_ars_process(ho, buf.ctypes.data, n, y1.ctypes.data, cap)
            n2 = r.ref_ars_process(hr, buf.ctypes.data, n, y2.ctypes.data, cap)
            assert n1 == n2 and y1[:n1].tobytes() == y2[:n2].tobytes(), k
            total += n1
    finally:
        o.oracle_ars_free(ho)
        r.ref_ars_free(hr)
    assert total > 50000


# ---- the reference's thread count ---------------------------------------------------------------------------------------
def reference_slices(n_threads, in_h, out_h):
    """(tasks, output lines per task) the reference's converter uses for n-threads on this host
    (video-converter.c:2466-2472: at most the online processors, then at least 200 lines per task; :3346: equal slices
    of ceil(out_h / tasks) lines - BGRA packs one line at a time)"""
    import os
    n = min(n_threads, os.sysconf("SC_NPROCESSORS_ONLN"))
    tallest = max(in_h, out_h)
    if tallest // n < 200:
        n = (tallest + 199) // 200
    n = max(n, 1)
    return n, -(-out_h // n)


@pytest.mark.ref
@pytest.mark.parametrize("case", [(1920, 1080, 3840, 2160, 0, 4), (1920, 1080, 3840, 2160, 0, 16), (3840, 2160, 1280, 720, 3, 4),
                                  (3840, 2160, 1280, 720, 3, 16)], ids=lambda c: "%dx%d-%dx%d-m%d-%dthreads" % c)
def test_reference_threads_change_bytes_at_slice_boundaries(case):
    """With n-threads > 1 the reference converts the frame in horizontal slices, one task each.  Every task owns its
    line caches (convert->pack_lines[i] and the caches before it; h_0 = i * lines_per_thread, video-converter.c:3350-3360) and starts them at its
    slice's first line, so on these shapes the bytes change from a slice boundary on; the tasks share no line state,
    and the shim's task pool is a plain pthread_create / pthread_join per task (oracle/refshim/shim.c).  The task count
    follows the host (reference_slices); with one task there is no boundary and the output is the single-threaded one.
    Every other test takes its expected bytes from the single-threaded reference (test below)."""
    iw, ih, ow, oh, method, threads = case
    tasks, lines = reference_slices(threads, ih, oh)
    frame = ob.nv12_random_frame(iw, ih, 1)
    r1, rn = ob.RefVcs(iw, ih, ow, oh, method, n_threads=1), ob.RefVcs(iw, ih, ow, oh, method, n_threads=threads)
    try:
        a, b = r1.convert(frame), rn.convert(frame)
    finally:
        r1.close()
        rn.close()
    bad = np.flatnonzero(a != b)
    if tasks == 1:
        assert bad.size == 0
        return
    assert bad.size > 0
    first_row = int(bad[0]) // (ow * 4)
    assert first_row > 0 and first_row % lines == 0, (tasks, lines, first_row)


def test_no_test_takes_bytes_from_a_threaded_reference():
    """RefVcs with n_threads other than 1 appears only in the tests of the thread count itself"""
    import os
    import re
    here = os.path.dirname(os.path.abspath(__file__))
    allowed = {("test_oracle_vs_ref.py", "test_reference_threads_equal_single_thread"),
               ("test_worstcase_ref.py", "test_reference_threads_change_bytes_at_slice_boundaries")}
    for name in sorted(os.listdir(here)):
        if not name.endswith(".py"):
            continue
        func = None
        for line in open(os.path.join(here, name)):
            m = re.match(r"def (\w+)", line)
            if m:
                func = m.group(1)
            for v in re.findall(r"RefVcs\(.*n_threads=([^,)]+)", line):
                assert v.strip() == "1" or (name, func) in allowed, (name, func, line.strip())
