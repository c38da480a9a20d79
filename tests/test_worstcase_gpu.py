"""Worst-case content on the H100 (tests/worstcase.py): frames whose windows sit at full scale on the side of each tap's
sign, and audio streams that drive chosen outputs past full scale, through every kernel the converter and the resampler
can launch, byte for byte against the oracle.  Noise never reaches these inputs; they are where a tap range, an
accumulator width or a saturating pack that is one stage early or late shows."""
import numpy as np
import pytest

import vcs_batch_cases as vb
import worstcase as wc
from oracle import bindings as ob
from test_vcs_batch_gpu import DevMem

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("row", vb.ROWS + wc.KNOB_ROWS, ids=lambda r: r.id)
def test_row_worst_case(cuda_device, row, monkeypatch):
    """every kernel of the batch rows (GRID_KERNELS and vcs_l2tc_kernel): batches of 2, 5 and 3 distinct worst-case
    frames on one handle; the handle reports the row's kernel and launch count"""
    from gstreamer_b200 import _lib
    h = wc.WorstHandle(_lib.lib, row, monkeypatch)
    try:
        vb.check_batches(h, DevMem(), (2, 5, 3), seed=100)
    finally:
        h.close()


# production shapes, NV12 -> BGRA: (id, size, method, kernel_name, variant, knob)
PROD = [
    ("4k-1080p-v2", (3840, 2160, 1920, 1080), 3, "vcs_lanczos2_v2_kernel", None, None),
    ("4k-1080p-v1", (3840, 2160, 1920, 1080), 3, "vcs_lanczos2_kernel", None, "B200_L2_V1=1"),
    ("4k-1080p-mma", (3840, 2160, 1920, 1080), 3, "vcs_l2mma_kernel", 6, None),
    ("4k-1080p-tc", (3840, 2160, 1920, 1080), 3, "vcs_l2tc_kernel", 7, None),
    ("4k-1080p-light", (3840, 2160, 1920, 1080), 1, "vcs_light_kernel", None, None),
    ("1080p-720p-ntap", (1920, 1080, 1280, 720), 3, "vcs_ntap_kernel", None, None),
    ("1080p-720p-mitchell", (1920, 1080, 1280, 720), 9, "vcs_ntap_kernel", None, None),
    ("1080p-720p-light", (1920, 1080, 1280, 720), 1, "vcs_light_kernel", None, None),
    ("1080p-4k-ntap", (1920, 1080, 3840, 2160), 3, "vcs_ntap_kernel", None, None),
    ("1080p-4k-light", (1920, 1080, 3840, 2160), 1, "vcs_light_kernel", None, None),
]


@pytest.mark.parametrize("case", PROD, ids=lambda c: c[0])
def test_production_shapes(cuda_device, case, monkeypatch):
    """NV12 -> BGRA at 4K -> 1080p (every 2:1 kernel), 1080p -> 720p and 1080p -> 4K: a batch of two different worst
    cases, one aimed at the taps and one random XOR-binary"""
    from gstreamer_b200 import _lib
    cid, size, method, name, variant, knob = case
    row = vb.Row(cid, "NV12", "BGRA", size, method, name, ("?",), variant=variant, knob=knob)
    h = wc.WorstHandle(_lib.lib, row, monkeypatch)
    try:
        vb.check_batches(h, DevMem(), (2,), seed=200)
    finally:
        h.close()


# ---- audio: every route the knobs reach ---------------------------------------------------------------------------------
# (format, (in, out, channels, quality), knobs): the persistent pipelines and their tile shapes, the FULL and small-channel
# kernels, the interpolated filter mode, the generic / direct kernels
ARS_CASES = [("F32", (48000, 44100, 256, 4), k) for k in
             (None, "B200_ARS_PIPE_V1=1", "B200_ARS_NOPIPE=1 B200_ARS_CPT=4", "B200_ARS_NOPIPE=1 B200_ARS_CPT=1",
              "B200_ARS_NOPIPE=1 B200_ARS_CB=64 B200_ARS_CPT=1", "B200_ARS_NOPIPE=1 B200_ARS_CB=32 B200_ARS_NO=16",
              "B200_ARS_NOPIPE=1 B200_ARS_NO=64", "B200_ARS_GRID=3", "B200_ARS_GENERIC=1")] + [
    ("S16", (48000, 44100, 256, 4), None), ("S16", (48000, 44100, 256, 4), "B200_ARS_GRID=3"),
    ("S16", (48000, 44100, 256, 4), "B200_ARS_NOPIPE=1"), ("S16", (48000, 44100, 2, 4), "B200_ARS_GENERIC=1"),
] + [(f, cfg, None) for f in ("F32", "S16", "S32", "F64")
     for cfg in ((48000, 44100, 2, 4), (96000, 44100, 3, 4), (44100, 48001, 2, 4), (48000, 44100, 70, 10))]


def _ars_id(c):
    f, (a, b, ch, q), k = c
    return "%s-%d-%d-%dch-q%d%s" % (f, a, b, ch, q, "" if k is None else "-" + k.replace(" ", "-"))


@pytest.mark.parametrize("case", ARS_CASES, ids=_ars_id)
def test_audio_worst_case(cuda_device, monkeypatch, case):
    import torch
    from gstreamer_b200.audio import CudaAudioResample
    fmt, cfg, knobs = case
    for kv in (knobs or "").split():
        monkeypatch.setenv(*kv.split("="))
    a, b, ch, q = cfg
    _, gfmt, dt, _ = ob.AUDIO_FORMATS[fmt]
    tdt = {np.float32: torch.float32, np.int16: torch.int16, np.int32: torch.int32, np.float64: torch.float64}[dt]
    for scale in sorted({wc.ars_scale(fmt, cfg), 1.0}):
        rs = CudaAudioResample(quality=q, format=gfmt)
        rs.set_caps(a, b, ch)

        def transform(chunk, n, cap):
            out = torch.full((cap * ch,), 7, dtype=tdt, device="cuda")
            ng = rs.transform(torch.from_numpy(chunk).cuda() if chunk is not None else None, n, out, cap)
            torch.cuda.synchronize()
            got = out.cpu().numpy().reshape(cap, ch)
            assert (got[ng:] == 7).all()
            return ng, got

        y, aims, full = wc.run_ars_case(transform, fmt, cfg, scale, seed=ch + q)
        if fmt in ("F32", "F64") or (scale < 1.0 and full):
            assert wc.check_saturation(y, aims, fmt) > 0
