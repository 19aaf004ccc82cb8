"""Shared helpers for the test-suite."""
from __future__ import annotations

from pathlib import Path

import numpy as np

import jxl_workload as wl
from libjxl_b200 import abi

GOLDEN = Path(__file__).resolve().parent / "golden"


class _Info:
    pass


class GoldenDump:
    """tests/golden/frame_small.npz viewed like an oracle.ref.FrameDump."""

    def __init__(self):
        z = np.load(GOLDEN / "frame_small.npz")
        self.z = z
        self.info = _Info()
        for k in z.files:
            if k.startswith("info_"):
                v = z[k]
                setattr(self.info, k[5:], v.tolist() if v.ndim else v.item())
        self.ac_strategy, self.raw_quant, self.sharpness = z["ac_strategy"], z["raw_quant"], z["sharpness"]
        self.ytox, self.ytob, self.dc = z["ytox"], z["ytob"], z["dc"]
        self.dequant, self.dequant_offsets, self.coeffs = z["dequant"], z["dequant_offsets"], z["coeffs"]
        self.taps = {k[4:]: z[k] for k in z.files if k.startswith("tap_")}
        self.decoded_default = z["decoded_default"]
        self.sigma_interior = z["sigma_interior"]


def golden_desc(**overrides) -> tuple[abi.FrameDesc, np.ndarray, GoldenDump]:
    from oracle import cpu as ocpu
    g = GoldenDump()
    return ocpu.desc_from_dump(g, **overrides), g.coeffs, g


def ulp_diff(a: np.ndarray, b: np.ndarray) -> int:
    """max distance in float32 ULPs (ordered-integer representation)."""
    ai = a.astype(np.float32).view(np.int32).astype(np.int64)
    bi = b.astype(np.float32).view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, np.int64(-2147483648) - ai, ai)
    bi = np.where(bi < 0, np.int64(-2147483648) - bi, bi)
    return int(np.abs(ai - bi).max())


TAP_MASKS = {"idct": 0, "gab_epf012": 15, "full": 31}


DC_STAGE_CASES = [(37, 21), (64, 48), (3, 3), (2, 9)]
DC_FACTORS = (3.1 / 4096, 1.7 / 512, 0.9 / 256)
DC_CFL = (0.0117, 0.0, 0.935)


# Every float scalar of jxlgpu_frame that the kernels read (FrameDev, filled in jxlgpu_frame_begin): the
# header fields of jxl_workload.HEADER_FIELDS plus the quantiser's global scale.  The sensitivity sweep of
# tests/test_gpu_header_parameters.py changes each entry (each channel separately) on its own.
SWEEP_FIELDS = ("inv_global_scale", "quant_scale") + wl.HEADER_FIELDS
# float scalars of jxlgpu_frame the sweep leaves to other tests, with where they are set away from defaults
SWEEP_EXEMPT = {"dc_factors": "DC stage: test_zz_dc_stage_gpu.py (support.DC_FACTORS)",
                "dc_cfl_factors": "DC stage: test_zz_dc_stage_gpu.py (support.DC_CFL)",
                "noise_lut": "noise: test_gpu_parity.py::test_noise_bit_exact (NOISE_LUT)"}
# swept again on a frame with noise: AddNoise reads the CfL base correlations and colour scale
NOISE_SWEEP = ("cfl_base_x", "cfl_base_b", "cfl_color_scale")


def sweep_entries(fields=SWEEP_FIELDS) -> list[tuple[str, int | None]]:
    """(field, channel or element index | None) for every scalar of `fields` (FrameDesc attribute names)."""
    sizes = {k: (n._length_ if hasattr(n, "_length_") else None) for k, n in abi.JxlGpuFrame._fields_}
    out = []
    for f in fields:
        n = 4 if f == "quant_biases" else sizes[f]
        out += [(f, None)] if n is None else [(f, i) for i in range(n)]
    return out


def perturbed(desc: abi.FrameDesc, field: str, idx: int | None) -> abi.FrameDesc:
    """A copy of `desc` (sharing its planes) with one scalar moved to another legal value: F16 fields by a
    factor 1.25 (0 -> 0.25), sharpness-LUT entries by + 0.5, the qm-scale multipliers one qm step, the colour factor by one, matrix entries
    by a factor 2 (exact, so still F16 x 255 / intensity_target)."""
    import copy
    d = copy.copy(desc)
    d._keep = []
    v = getattr(desc, field)
    old = float(v if idx is None else v[idx])
    if field == "cfl_color_scale":
        new = float(np.float32(1.0) / np.float32(round(1.0 / old) + 1))
    elif field in ("x_dm_multiplier", "b_dm_multiplier", "inv_global_scale", "quant_scale", "opsin_biases_cbrt"):
        new = float(np.float32(old * 1.25))
    elif field == "inverse_opsin_matrix":
        new = 2.0 * old
    elif field == "epf_sharp_lut":     # + 0.5: small entries leave EPF skipped (sigma below kMinSigma) either way
        new = float(wl.f16(old + 0.5))
    else:
        new = float(wl.f16(old * 1.25 if old else 0.25))
    assert new != old, (field, idx, old)
    if idx is None:
        setattr(d, field, new)
    else:
        t = list(v)
        t[idx] = new
        setattr(d, field, tuple(t))
    return d


def header_frame(w: int, h: int, seed: int, hdr, gab: int = 1, epf_iters: int = 3, ac_type: int = abi.AC_INT16):
    """A synthetic frame that exercises every header field: EPF engaged on most blocks with every sharpness
    value 0..7 (so every epf_sharp_lut entry is read), quantisers 1..3 and coefficients in -3..3 (both branches
    of AdjustQuantBias), and the non-default header `hdr` (jxl_workload.header_params name or seed)."""
    desc, coeffs = wl.synthetic_frame(w, h, seed=seed, gab=gab, epf_iters=epf_iters, ac_type=ac_type, density=0.08)
    rng = np.random.default_rng(seed + 7)
    desc.raw_quant = np.where(desc.raw_quant > 0, rng.integers(1, 4, desc.raw_quant.shape), 0).astype(np.int32)
    desc.epf_sharpness = rng.integers(0, 8, desc.epf_sharpness.shape).astype(np.uint8)
    coeffs = np.clip(coeffs, -3, 3)
    wl.apply_header(desc, wl.header_params(hdr))
    return desc, coeffs


def dc_stage_input(xs: int, ys: int) -> np.ndarray:
    """Seeded quantised DC planes (X, Y, B): smooth gradients (adaptive smoothing engages) with one busy
    quadrant (it must switch itself off there)."""
    rng = np.random.default_rng(1000 * xs + ys)
    yy, xx = np.mgrid[0:ys, 0:xs]
    q = np.stack([np.round(20 * np.sin(xx / 17 + c) + 15 * np.cos(yy / 23 + c) + rng.random((ys, xs)) * 1.2)
                  for c in range(3)]).astype(np.int32)
    q[:, ys // 2:, xs // 2:] += rng.integers(-40, 40, (3, ys - ys // 2, xs - xs // 2))
    return q
