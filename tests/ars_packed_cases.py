"""Shared by the packed-format resampler tests, the golden generator and the benchmark tool: the sample formats
cudaaudioresample unpacks (every GstAudioFormat but S16LE, S32LE, F32LE and F64LE), test signals in them, and ctypes
bindings of the two checkers of those formats — oracle_ars_*_packed (oracle/oracle_audio_packed.c) and the reference's
own converter steps (oracle/refshim/refdrv_audio_packed.c, built by oracle/packed.mk into oracle/_ref/)."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PACKED_SO = os.path.join(ROOT, "oracle", "_ref", "libgstref_packed.so")

# name -> (GstAudioFormat value, bytes per sample in a buffer, bytes between samples, depth, signed, big-endian, float)
FORMATS = {
    "S8": (2, 1, 1, 8, True, False, False), "U8": (3, 1, 1, 8, False, False, False),
    "S16BE": (5, 2, 2, 16, True, True, False), "U16LE": (6, 2, 2, 16, False, False, False),
    "U16BE": (7, 2, 2, 16, False, True, False),
    "S24_32LE": (8, 4, 4, 24, True, False, False), "S24_32BE": (9, 4, 4, 24, True, True, False),
    "U24_32LE": (10, 4, 4, 24, False, False, False), "U24_32BE": (11, 4, 4, 24, False, True, False),
    "S32BE": (13, 4, 4, 32, True, True, False), "U32LE": (14, 4, 4, 32, False, False, False),
    "U32BE": (15, 4, 4, 32, False, True, False),
    "S24LE": (16, 3, 3, 24, True, False, False), "S24BE": (17, 3, 3, 24, True, True, False),
    "U24LE": (18, 3, 3, 24, False, False, False), "U24BE": (19, 3, 3, 24, False, True, False),
    "S20LE": (20, 3, 3, 20, True, False, False), "S20BE": (21, 3, 3, 20, True, True, False),
    "U20LE": (22, 3, 3, 20, False, False, False), "U20BE": (23, 3, 3, 20, False, True, False),
    "S18LE": (24, 3, 3, 18, True, False, False), "S18BE": (25, 3, 3, 18, True, True, False),
    "U18LE": (26, 3, 3, 18, False, False, False), "U18BE": (27, 3, 3, 18, False, True, False),
    "F32BE": (29, 4, 4, 32, True, True, True), "F64BE": (31, 8, 8, 64, True, True, True),
    "S20_32LE": (32, 4, 3, 20, True, False, False), "S20_32BE": (33, 4, 3, 20, True, True, False),
    "U20_32LE": (34, 4, 3, 20, False, False, False), "U20_32BE": (35, 4, 3, 20, False, True, False),
}
NAMES = list(FORMATS)
# one representative of each way a format is stored: the GPU test and the route fixture use these
CLASSES = ["U8", "S16BE", "S24_32LE", "U32BE", "S24LE", "S20BE", "F32BE", "F64BE", "S20_32LE"]

# the element's resample-method / sinc-filter-mode / sinc-filter-interpolation sets of the emulated kernel tests
OPTS = [("kaiser", "auto", "cubic"), ("blackman-nuttall", "auto", "cubic"), ("kaiser", "full", "none"),
        ("kaiser", "interpolated", "cubic"), ("blackman-nuttall", "full", "none"), ("kaiser", "interpolated", "none"),
        ("kaiser", "full", "linear"), ("kaiser", "interpolated", "linear"), ("blackman-nuttall", "interpolated", "linear"),
        ("nearest", "auto", "cubic"), ("linear", "auto", "cubic"), ("cubic", "auto", "cubic")]
# the reference's enum values (oracle_ars_new_opts, ref_ars_new_opts)
REF_METHOD = {"nearest": 0, "linear": 1, "cubic": 2, "blackman-nuttall": 3, "kaiser": 4}
REF_MODE = {"interpolated": 0, "full": 1, "auto": 2}
REF_INTERP = {"none": 0, "linear": 1, "cubic": 2}


def width(fmt):
    return FORMATS[fmt][1]


def n_bytes(fmt, frames, ch):
    return frames * ch * width(fmt)


def packed_signal(rng, n, ch, fmt):
    """n frames x ch channels of fmt as bytes: integer formats random codes with runs of the extreme codes (full scale
    both ways, so the saturating bias and the sign flip are reached), float formats noise with +-1, +-0, denormals and
    the largest finite values; bytes between the samples of the 20-bit _32 formats are random"""
    _, w, step, depth, signed, big, is_float = FORMATS[fmt]
    buf = np.frombuffer(rng.integers(0, 256, n * ch * w, dtype=np.uint8).tobytes(), dtype=np.uint8).copy()
    k = n * ch
    if is_float:
        big_val = 3.4028234663852886e38 if w == 4 else 1e300
        tiny = 1e-40 if w == 4 else 1e-310
        v = rng.standard_normal(k) * 0.5
        pick = rng.random(k)
        for lo, hi, val in [(0.0, 0.02, 1.0), (0.02, 0.04, -1.0), (0.04, 0.05, 0.0), (0.05, 0.06, -0.0), (0.06, 0.07, tiny),
                            (0.07, 0.08, -tiny), (0.08, 0.09, big_val), (0.09, 0.1, -big_val)]:
            v[(pick >= lo) & (pick < hi)] = val
        dt = (">f4" if big else "<f4") if w == 4 else (">f8" if big else "<f8")
        return np.frombuffer(v.astype(dt).tobytes(), dtype=np.uint8).copy()
    codes = rng.integers(0, 1 << depth, k, dtype=np.uint64)
    top = (1 << depth) - 1 if not signed else (1 << (depth - 1)) - 1
    bottom = 0 if not signed else 1 << (depth - 1)
    pick = rng.random(k)
    codes[pick < 0.1] = top
    codes[(pick >= 0.1) & (pick < 0.2)] = bottom
    # runs of one extreme: whole windows at full scale
    for s in range(0, k, 97):
        codes[s:s + 9 * ch] = top if (s // 97) % 2 else bottom
    order = range(step - 1, -1, -1) if big else range(step)
    for j, b in enumerate(order):
        buf[np.arange(k) * step + b] = ((codes >> np.uint64(8 * j)) & np.uint64(0xFF)).astype(np.uint8)
    return buf


_oracle = None
_ref = None


def oracle():
    global _oracle
    if _oracle is None:
        from oracle import bindings as ob
        o = ob.oracle()
        P = C.c_void_p
        o.oracle_ars_new_packed.restype = P
        o.oracle_ars_new_packed.argtypes = [C.c_int] * 8
        o.oracle_ars_packed_resampler.restype = P
        o.oracle_ars_packed_resampler.argtypes = [P]
        o.oracle_ars_process_packed.restype = C.c_size_t
        o.oracle_ars_process_packed.argtypes = [P, P, C.c_size_t, P, C.c_size_t]
        o.oracle_ars_free_packed.argtypes = [P]
        o.oracle_ars_packed_width.argtypes = [C.c_int]
        _oracle = o
    return _oracle


def have_ref():
    return os.path.exists(REF_PACKED_SO)


def ref():
    global _ref
    if _ref is None:
        from oracle import bindings as ob
        ob.ref()                               # argument types of ref_ars_update / _get_out_frames / _reset
        r = C.CDLL(REF_PACKED_SO)
        P = C.c_void_p
        r.ref_ars_new_packed.restype = P
        r.ref_ars_new_packed.argtypes = [C.c_int] * 8
        r.ref_ars_packed_resampler.restype = P
        r.ref_ars_packed_resampler.argtypes = [P]
        r.ref_ars_process_packed.restype = C.c_size_t
        r.ref_ars_process_packed.argtypes = [P, P, C.c_size_t, P, C.c_size_t]
        r.ref_ars_free_packed.argtypes = [P]
        _ref = r
    return _ref


class OraclePacked:
    """one oracle stream of a packed format (the reference's enum values in opts)"""

    def __init__(self, a, b, ch, q, fmt, opts=OPTS[0]):
        m, mo, it = opts
        self.o, self.ch, self.fmt = oracle(), ch, fmt
        self.h = self.o.oracle_ars_new_packed(a, b, ch, q, FORMATS[fmt][0], REF_METHOD[m], REF_MODE[mo], REF_INTERP[it])
        assert self.h

    def process(self, x, n, cap, fill=7):
        out = np.full(n_bytes(self.fmt, cap, self.ch), fill, dtype=np.uint8)
        got = self.o.oracle_ars_process_packed(self.h, x.ctypes.data if x is not None else None, n, out.ctypes.data, cap)
        return got, out

    def resampler(self):
        return self.o.oracle_ars_packed_resampler(self.h)

    def free(self):
        self.o.oracle_ars_free_packed(self.h)


def config(lib_mod, a, b, ch, q, fmt, opts=OPTS[0]):
    """b200_ars_config for fmt (a FORMATS name or a b200 format value)"""
    from gstreamer_b200 import _lib
    from gstreamer_b200.audio import CudaAudioResample as A
    m, mo, it = opts
    cfg = _lib.ArsConfigC()
    cfg.in_rate, cfg.out_rate, cfg.channels, cfg.quality = a, b, ch, q
    cfg.format = FORMATS[fmt][0] if isinstance(fmt, str) else fmt
    cfg.resample_method, cfg.sinc_filter_mode, cfg.sinc_filter_interpolation = A.METHODS[m], A.FILTER_MODES[mo], A.INTERPOLATIONS[it]
    return cfg
