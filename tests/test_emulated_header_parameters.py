"""The kernels at non-default frame-header parameters under the SIMT emulation of tests/emu (no GPU): a small
subset of tests/test_gpu_header_parameters.py on the two-kernel and the fused context, bit-exact against the
oracle, and the check that the GPU file's sensitivity sweep covers every float scalar of jxlgpu_frame."""
import ctypes as C

import numpy as np
import pytest

from libjxl_b200 import abi, pipeline
from tests import support


@pytest.fixture(scope="module", params=["two-kernel", "fused"])
def emu_pipe(request):
    """The emulated library (tests/emu) in place of libjxl_b200.so, one context per decode path."""
    import os
    from tests.emu import build_emu
    so = build_emu.build()
    saved = pipeline._lib
    pipeline._lib = pipeline.bind(C.CDLL(str(so)))
    old = os.environ.get("JXLGPU_FUSED")
    os.environ["JXLGPU_FUSED"] = "1" if request.param == "fused" else "0"
    try:
        p = pipeline.TransformPipeline(device=0, num_host_threads=2)
        yield p
        p.close()
    finally:
        pipeline._lib = saved
        if old is None:
            os.environ.pop("JXLGPU_FUSED", None)
        else:
            os.environ["JXLGPU_FUSED"] = old


def oracle(desc, coeffs):
    from oracle import cpu
    return cpu.render_frame(desc, coeffs, rcp_mode=0)


# (header set, path): strip kernel (Gaborish + EPF 1 + 2, a chain the fused kernel runs too), the tile kernel
# (explicit chain outside the production set, 8-bit sRGB, int32), noise (AddNoise reads the CfL base)
CASES = [("dim80", "strip"), ("pq10000", "tile"), ("edges", "noise")]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("hdr,path", CASES, ids=[c[1] for c in CASES])
def test_emulated_header_sets(emu_pipe, hdr, path):
    from tests.test_emulated_cuda import NOISE_LUT
    ac = abi.AC_INT32 if path == "tile" else abi.AC_INT16
    desc, coeffs = support.header_frame(203, 137, seed=len(path), hdr=hdr, gab=1,
                                        epf_iters=1 if path == "noise" else 2, ac_type=ac)
    if path == "tile":
        desc.out_format = abi.OUT_RGB_U8
        desc.stage_mask = abi.STAGE_EXPLICIT | abi.STAGE_GAB | abi.STAGE_EPF2 | abi.STAGE_XYB | abi.STAGE_SRGB
    if path == "noise":
        desc.noise, desc.noise_lut = 1, NOISE_LUT
        desc.visible_frame_index, desc.nonvisible_frame_index = 2, 1
    want = oracle(desc, coeffs)
    got = emu_pipe.decode_frame(desc, coeffs)
    assert got.shape == want.shape and np.array_equal(got, want), f"{path} at header {hdr}"


def test_sweep_covers_every_frame_scalar():
    """Every float scalar of jxlgpu_frame is in the GPU sensitivity sweep (support.SWEEP_FIELDS) or named in
    support.SWEEP_EXEMPT with the test that sets it away from its default: a header field added to the ABI
    without a sweep entry fails here."""
    floats = {n for n, t in abi.JxlGpuFrame._fields_ if t is C.c_float or getattr(t, "_type_", None) is C.c_float}
    assert floats == set(support.SWEEP_FIELDS) | set(support.SWEEP_EXEMPT)
    assert set(support.NOISE_SWEEP) <= set(support.SWEEP_FIELDS)
    entries = support.sweep_entries()
    assert len(entries) == len(set(entries)) == 47
