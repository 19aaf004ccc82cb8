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


K_MIN_SIGMA = np.float32(-3.90524291751269967465540850526868)   # epf.h: blocks with 1/sigma below it skip the EPF
EPF_STAGES = abi.STAGE_EPF0 | abi.STAGE_EPF1 | abi.STAGE_EPF2


def block_quant(desc: abi.FrameDesc) -> np.ndarray:
    """raw_quant of the varblock covering each 8x8 block (raw_quant itself is defined on first blocks only)."""
    acs = desc.ac_strategy
    out = np.zeros(acs.shape, np.int64)
    first = (acs & 1) == 1
    for s in range(27):
        ys, xs = np.nonzero(first & ((acs >> 1) == s))
        for iy in range(abi.COVERED_Y[s]):
            for ix in range(abi.COVERED_X[s]):
                out[ys + iy, xs + ix] = desc.raw_quant[ys, xs]
    return out


def epf_frame(w: int, h: int, seed: int, gab: int = 1, epf_iters: int = 3, ac_type: int = abi.AC_INT16, hdr=None,
              strategies: str = "all"):
    """A synthetic frame on which the EPF does real work everywhere: about half of the varblocks get a quantiser
    1..4, the rest 40..256 (EPF skipped), every block a sharpness 0..7, so engaged and skipped blocks mix inside
    every block row of every 256-column strip (the strip kernel's block permutation is not the identity).  Varblocks
    32 or more columns wide always get a quantiser 1..2, else one large transform of high quantiser would leave a
    whole strip block row unfiltered.  Small, clipped coefficients keep the SADs small enough that many EPF weights lie
    strictly inside (0, 1).  `hdr`: a jxl_workload.header_params name or seed."""
    desc, coeffs = wl.synthetic_frame(w, h, seed=seed, strategies=strategies, gab=gab, epf_iters=epf_iters,
                                      ac_type=ac_type, density=0.08)
    rng = np.random.default_rng(seed + 4242)
    shape = desc.raw_quant.shape
    acs = desc.ac_strategy
    wide = np.array([abi.COVERED_X[s] >= 4 for s in range(27)])[acs >> 1]
    q = np.where(rng.random(shape) < 0.5, rng.integers(1, 5, shape), rng.integers(40, 257, shape))
    q = np.where(wide, rng.integers(1, 3, shape), q)
    desc.raw_quant = np.where((acs & 1) == 1, q, 0).astype(np.int32)
    desc.epf_sharpness = rng.integers(0, 8, shape).astype(np.uint8)
    coeffs = np.clip(coeffs, -3, 3)
    # a flat block is a fixed point of the EPF and a block edge of synthetic_frame's DC noise zeroes every weight
    # across it: a tenth of the DC noise and 1/25 of the AC amplitude leave SADs where the weights are neither
    mean = desc.dc.mean(axis=(1, 2), keepdims=True)
    desc.dc = (mean + np.float32(0.1) * (desc.dc - mean)).astype(np.float32)
    desc.dequant = (desc.dequant * np.float32(0.04)).astype(np.float32)
    if hdr is not None:
        wl.apply_header(desc, wl.header_params(hdr))
    eng = epf_engaged_blocks(desc)
    frac = eng.mean()
    assert 0.2 <= frac <= 0.75, frac
    # every block row of every full 32-block strip holds engaged and skipped blocks
    xb = desc.xsize_blocks
    for x0 in range(0, xb - 31, 32):
        part = eng[:, x0:x0 + 32]
        assert part.any(1).all() and (~part).any(1).all(), (w, h, seed, x0)
    return desc, coeffs


def epf_engaged_blocks(desc: abi.FrameDesc) -> np.ndarray:
    """(ysize_blocks, xsize_blocks) bool: blocks whose inverse sigma (the oracle's ComputeSigma) engages the EPF."""
    from oracle import cpu as ocpu
    return ~(ocpu.compute_sigma(desc)[2:-2, 2:-2] < K_MIN_SIGMA)


def without_epf(desc: abi.FrameDesc) -> abi.FrameDesc:
    """The same stage chain with every EPF pass taken out."""
    import dataclasses
    if desc.stage_mask & abi.STAGE_EXPLICIT:
        return dataclasses.replace(desc, stage_mask=desc.stage_mask & ~EPF_STAGES)
    return dataclasses.replace(desc, epf_iters=0)


def changed_pixels(a: np.ndarray, b: np.ndarray, planar: bool) -> np.ndarray:
    """(H, W) bool: pixels where any channel of two renders differs."""
    d = a != b
    return d.any(0) if planar else d.reshape(d.shape[0], d.shape[1], -1).any(2)


def epf_coverage(desc: abi.FrameDesc, coeffs: np.ndarray, render=None, with_epf: np.ndarray | None = None) -> np.ndarray:
    """The oracle's changed-pixel mask of the EPF: the frame's chain against the same chain without EPF passes.
    `render(desc)` renders through the oracle (a caching one, say); `with_epf`: the chain's image if at hand."""
    if render is None:
        from oracle import cpu as ocpu
        render = lambda d: ocpu.render_frame(d, coeffs, rcp_mode=0)   # noqa: E731
    a = with_epf if with_epf is not None else render(desc)
    return changed_pixels(a, render(without_epf(desc)), desc.out_format == abi.OUT_PLANAR_F32)


def _every_window(any_: np.ndarray, n: int) -> bool:
    """True if every window of n consecutive entries (the whole array if shorter) holds a True."""
    if any_.size <= n:
        return bool(any_.any())
    c = np.concatenate([[0], np.cumsum(any_)])
    return bool((c[n:] - c[:-n] > 0).all())


def assert_epf_coverage(mask: np.ndarray, what: str, boundary_min: int = 200, band_rows=None) -> None:
    """Every group-row boundary (and the `band_rows` boundaries) +-7 rows holds at least `boundary_min` changed
    pixels; every 64-row window (the strip kernel's shortest row segment) and every 240-column window (a fused-kernel
    strip) holds one.  Prints the figures."""
    h, w = mask.shape
    bounds = sorted(set(range(abi.GROUP_DIM, h, abi.GROUP_DIM)) | set(band_rows or ()))
    counts = [int(mask[max(0, y - 7):y + 7].sum()) for y in bounds]
    rows, cols = mask.any(1), mask.any(0)
    print(f"EPF coverage {what}: {mask.mean():.2%} of pixels changed; +-7 rows around {len(bounds)} boundaries: "
          f"min {min(counts, default=0)} changed; 64-row windows all hit: {_every_window(rows, 64)}; "
          f"240-column windows all hit: {_every_window(cols, 240)}")
    assert all(c >= boundary_min for c in counts), (what, list(zip(bounds, counts)))
    assert _every_window(rows, 64), what
    assert _every_window(cols, 240), what


def decoy_frame(desc: abi.FrameDesc, seed: int):
    """A frame of the same geometry, ac_type, chain and output as `desc` with other coefficients, a DC offset and
    the EPF engaged on every block.  Rendered on a context just before `desc`, it leaves every device buffer full of
    values that are wrong for `desc`: a kernel that reads a row before it is written shows it in the pixels."""
    import dataclasses
    d, coeffs = wl.synthetic_frame(desc.xsize, desc.ysize, seed=seed, gab=desc.gab, epf_iters=3, ac_type=desc.ac_type,
                                   density=0.05)
    d = dataclasses.replace(desc, ac_strategy=d.ac_strategy, dc=d.dc + np.float32(0.05), ytox=d.ytox, ytob=d.ytob,
                            raw_quant=np.where(d.raw_quant > 0, 1, 0).astype(np.int32),
                            epf_sharpness=np.full_like(d.epf_sharpness, 7))
    return d, np.clip(coeffs, -2, 2)


def assert_decoy_differs(decoy_px: np.ndarray, want: np.ndarray, planar: bool, min_frac: float = 0.99) -> None:
    frac = changed_pixels(decoy_px, want, planar).mean()
    assert frac >= min_frac, f"the decoy matches the target on {1 - frac:.2%} of the pixels"


def dc_stage_input(xs: int, ys: int) -> np.ndarray:
    """Seeded quantised DC planes (X, Y, B): smooth gradients (adaptive smoothing engages) with one busy
    quadrant (it must switch itself off there)."""
    rng = np.random.default_rng(1000 * xs + ys)
    yy, xx = np.mgrid[0:ys, 0:xs]
    q = np.stack([np.round(20 * np.sin(xx / 17 + c) + 15 * np.cos(yy / 23 + c) + rng.random((ys, xs)) * 1.2)
                  for c in range(3)]).astype(np.int32)
    q[:, ys // 2:, xs // 2:] += rng.integers(-40, 40, (3, ys - ys // 2, xs - xs // 2))
    return q
