"""ctypes binding of libb200dsp.so (the C-ABI declared in include/b200dsp.h).

The library is the product; this module only loads it and declares signatures.  There
is no CPU fallback: if the shared object is missing the import fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200dsp.so")

MAX_PLANES = 4
VCS_MAX_BATCH = 64
COMP_MAX_PADS = 64


class B200Error(RuntimeError):
    def __init__(self, status, where=""):
        self.status = status
        msg = lib.b200_strerror(status).decode()
        if status == -4:
            msg += ": " + lib.b200_last_cuda_error().decode()
        super().__init__(f"{where}: {msg} ({status})" if where else f"{msg} ({status})")


class VideoInfoC(C.Structure):
    _fields_ = [("format", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("stride", C.c_int32 * MAX_PLANES), ("offset", C.c_uint64 * MAX_PLANES),
                ("color_matrix", C.c_int32), ("color_range", C.c_int32), ("chroma_site", C.c_int32)]


class VcsConfigC(C.Structure):
    _fields_ = [("method", C.c_int32), ("envelope", C.c_double), ("sharpness", C.c_double),
                ("sharpen", C.c_double), ("dest_x", C.c_int32), ("dest_y", C.c_int32), ("dest_width", C.c_int32),
                ("dest_height", C.c_int32), ("border_argb", C.c_uint32), ("fill_border", C.c_int32),
                ("reserved", C.c_int32 * 2)]


class VcsPlanInfoC(C.Structure):
    _fields_ = [("h_taps", C.c_int32), ("v_taps", C.c_int32), ("h_first", C.c_int32),
                ("matrix_first", C.c_int32), ("p", C.c_int32 * 5), ("tile_w", C.c_int32),
                ("tile_h", C.c_int32), ("smem_bytes", C.c_int32), ("kernel_variant", C.c_int32),
                ("n_launches_per_convert", C.c_int32)]


class CompPadC(C.Structure):
    _fields_ = [("data", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32),
                ("stride", C.c_int32), ("xpos", C.c_int32), ("ypos", C.c_int32),
                ("alpha", C.c_double), ("op", C.c_int32), ("reserved", C.c_int32)]


class CompPadYuvC(C.Structure):
    _fields_ = [("data", C.c_void_p), ("info", VideoInfoC), ("xpos", C.c_int32), ("ypos", C.c_int32),
                ("alpha", C.c_double), ("op", C.c_int32), ("reserved", C.c_int32)]


class CompPadConvertC(C.Structure):
    _fields_ = [("data", C.c_void_p), ("info", VideoInfoC), ("conv", C.c_void_p), ("xpos", C.c_int32), ("ypos", C.c_int32),
                ("alpha", C.c_double), ("op", C.c_int32), ("reserved", C.c_int32)]


class ArsConfigC(C.Structure):
    _fields_ = [("in_rate", C.c_int32), ("out_rate", C.c_int32), ("channels", C.c_int32),
                ("quality", C.c_int32), ("format", C.c_int32), ("resample_method", C.c_int32),
                ("sinc_filter_mode", C.c_int32), ("sinc_filter_interpolation", C.c_int32), ("reserved", C.c_int32 * 4)]


class ArsPlanInfoC(C.Structure):
    _fields_ = [("n_taps", C.c_int32), ("n_phases", C.c_int32), ("in_step", C.c_int32),
                ("out_step", C.c_int32), ("filter_mode", C.c_int32), ("oversample", C.c_int32)]


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with ./build.sh (or __graft_entry__.build()). "
        "gstreamer_b200 has no CPU fallback.")

lib = C.CDLL(LIB_PATH)

_P = C.c_void_p
_SIGS = {
    "b200_strerror": (C.c_char_p, [C.c_int]),
    "b200_last_cuda_error": (C.c_char_p, []),
    "b200_version": (C.c_int, []),
    "b200_device_count": (C.c_int, []),
    "b200_host_alloc": (C.c_int, [C.c_size_t, C.POINTER(_P)]),
    "b200_host_free": (C.c_int, [_P]),
    "b200_host_alloc_near": (C.c_int, [C.c_int, C.c_size_t, C.POINTER(_P)]),
    "b200_device_numa_node": (C.c_int, [C.c_int]),
    "b200_video_info_set_format": (C.c_int, [C.POINTER(VideoInfoC), C.c_int, C.c_int, C.c_int]),
    "b200_video_info_size": (C.c_size_t, [C.POINTER(VideoInfoC)]),
    "b200_vcs_config_init": (None, [C.POINTER(VcsConfigC)]),
    "b200_vcs_create": (C.c_int, [C.POINTER(VideoInfoC), C.POINTER(VideoInfoC), C.POINTER(VcsConfigC),
                                  C.c_int, C.POINTER(_P)]),
    "b200_vcs_destroy": (None, [_P]),
    "b200_vcs_convert": (C.c_int, [_P, _P, _P, _P]),
    "b200_vcs_convert_batch": (C.c_int, [_P, C.c_int, C.POINTER(_P), C.POINTER(_P), _P]),
    "b200_vcs_convert_host": (C.c_int, [_P, C.c_int, C.POINTER(_P), C.POINTER(_P)]),
    "b200_vcs_copy_probe": (C.c_int, [_P, C.c_int, C.POINTER(_P), C.POINTER(_P)]),
    "b200_vcs_get_plan_info": (C.c_int, [_P, C.POINTER(VcsPlanInfoC)]),
    "b200_vcs_get_taps": (C.c_int, [_P, C.c_int, _P, _P, C.c_size_t, C.c_size_t]),
    "b200_vcs_get_matrix": (C.c_int, [_P, _P]),
    "b200_vcs_get_chroma_plan": (C.c_int, [_P, _P, C.c_size_t]),
    "b200_vcs_set_kernel_variant": (C.c_int, [_P, C.c_int]),
    "b200_vcs_kernel_name": (C.c_char_p, [_P]),
    "b200_comp_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "b200_comp_destroy": (None, [_P]),
    "b200_comp_blend": (C.c_int, [_P, _P, C.c_int32, C.c_int, C.POINTER(CompPadC), C.c_int, _P]),
    "b200_comp_blend_host_submit": (C.c_int, [_P, _P, C.c_int32, C.c_int, C.POINTER(CompPadC), C.c_int]),
    "b200_comp_blend_host_wait": (C.c_int, [_P, C.c_int]),
    "b200_comp_blend_yuv_host_submit": (C.c_int, [_P, _P, C.POINTER(VideoInfoC), C.c_int, C.POINTER(CompPadYuvC), C.c_int]),
    "b200_comp_blend_yuv_host": (C.c_int, [_P, _P, C.POINTER(VideoInfoC), C.c_int, C.POINTER(CompPadYuvC), C.c_int]),
    "b200_comp_blend_host": (C.c_int, [_P, _P, C.c_int32, C.c_int, C.POINTER(CompPadC), C.c_int]),
    "b200_comp_blend_yuv": (C.c_int, [_P, _P, C.POINTER(VideoInfoC), C.c_int, C.POINTER(CompPadYuvC), C.c_int, _P]),
    "b200_comp_blend_convert": (C.c_int, [_P, _P, C.POINTER(VideoInfoC), C.c_int, C.POINTER(CompPadConvertC), C.c_int, _P]),
    "b200_ars_create": (C.c_int, [C.POINTER(ArsConfigC), C.c_int, C.POINTER(_P)]),
    "b200_ars_destroy": (None, [_P]),
    "b200_ars_reset": (C.c_int, [_P]),
    "b200_ars_update": (C.c_int, [_P, C.c_int, C.c_int]),
    "b200_ars_get_out_frames": (C.c_size_t, [_P, C.c_size_t]),
    "b200_ars_get_in_frames": (C.c_size_t, [_P, C.c_size_t]),
    "b200_ars_get_max_latency": (C.c_size_t, [_P]),
    "b200_ars_process": (C.c_int, [_P, _P, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_size_t), _P]),
    "b200_ars_process_host_submit": (C.c_int, [_P, _P, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200_ars_process_host_wait": (C.c_int, [_P, C.c_int]),
    "b200_ars_process_host": (C.c_int, [_P, _P, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200_ars_get_plan_info": (C.c_int, [_P, C.POINTER(ArsPlanInfoC)]),
    "b200_ars_get_phase_taps": (C.c_int, [_P, C.c_int, _P, C.c_size_t]),
}

#: every symbol include/b200dsp.h declares; tests assert the .so exports all of them
EXPORTED_SYMBOLS = tuple(_SIGS)

_missing = []
for _name, (_res, _args) in _SIGS.items():
    try:
        _fn = getattr(lib, _name)
    except AttributeError:
        _missing.append(_name)
        continue
    _fn.restype = _res
    _fn.argtypes = _args
MISSING_SYMBOLS = tuple(_missing)


def check(status, where=""):
    if status < 0:
        raise B200Error(status, where)
    return status
