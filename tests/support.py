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


# ---- upsampling and noise ----

# A strength LUT of legal values (NoiseParams: 10-bit codes k / 1024, k <= 1023) that spans 0 .. 1023/1024 and is
# not monotone, so every segment of StrengthEvalLut interpolates between different values.
NOISE_LUT_WIDE = tuple(k / 1024 for k in (96, 1023, 410, 0, 700, 255, 880, 512))
UPS_WEIGHT_COUNT = {2: 15, 4: 55, 8: 210}


def default_upsampling_weights(n: int) -> np.ndarray:
    return np.load(GOLDEN / "upsampling_weights.npz")[f"weights{n}"]


def custom_upsampling_weights(n: int, seed: int) -> np.ndarray:
    """Random F16 weights of factor n (CustomTransformData::upsampling{n}_weights): the defaults scaled by 0.4..1.6
    with noise added and a tenth of the signs flipped, so no two entries of the triangular layout are related."""
    rng = np.random.default_rng(seed)
    d = default_upsampling_weights(n).astype(np.float64)
    w = d * rng.uniform(0.4, 1.6, d.size) + rng.normal(0, 0.02, d.size)
    w = np.where(rng.random(d.size) < 0.1, -w, w)
    return wl.f16(w)


def filter_mask(desc: abi.FrameDesc) -> int:
    """The filter stages (Gaborish, EPF passes) of the frame's chain as stage-mask bits."""
    if desc.stage_mask & abi.STAGE_EXPLICIT:
        return desc.stage_mask & 15
    return ((abi.STAGE_GAB if desc.gab else 0) | (abi.STAGE_EPF0 if desc.epf_iters >= 3 else 0) |
            (abi.STAGE_EPF1 if desc.epf_iters >= 1 else 0) | (abi.STAGE_EPF2 if desc.epf_iters >= 2 else 0))


def pre_upsampling_desc(desc: abi.FrameDesc) -> abi.FrameDesc:
    """The same frame cut after its filters: planar XYB at the coded size, without upsampling and noise."""
    import dataclasses
    return dataclasses.replace(desc, upsampling=0, upsampling_weights=None, xsize_upsampled=0, ysize_upsampled=0,
                               noise=0, stage_mask=abi.STAGE_EXPLICIT | filter_mask(desc),
                               out_format=abi.OUT_PLANAR_F32)


def out_size(desc: abi.FrameDesc) -> tuple[int, int]:
    n = desc.upsampling if desc.upsampling > 1 else 1
    return (desc.xsize_upsampled or n * desc.xsize, desc.ysize_upsampled or n * desc.ysize) if n > 1 \
        else (desc.xsize, desc.ysize)


def ups_noise_frame(n: int, w: int, h: int, seed: int, weights: str = "custom", lut=NOISE_LUT_WIDE, noise: bool = True,
                    hdr=None, gab: int = 1, epf_iters: int = 1, fmt: int = abi.OUT_RGB_F32, srgb: int = 0,
                    ac_type: int = abi.AC_INT16, frame_index=(3, 1)):
    """A frame that drives the upsampling and the noise into all their branches.  n: 1 (noise only), 2, 4 or 8;
    the output is n*w - (n-1) x n*h - 1 (ragged).  Per 8x8 block the Y DC is drawn from one of three ranges: 1.5..3
    (AddNoise's strength saturates), -0.6..-0.05 (below X: negative input, clamped to the LUT's start) or 0..1.5
    (every LUT segment); independent block DCs make hard edges, where the upsampler's window clamp engages.
    `weights`: "custom" (random F16, custom_upsampling_weights) or "default"; `hdr`: a jxl_workload.header_params
    name or seed (header_frame)."""
    if hdr is not None:
        desc, coeffs = header_frame(w, h, seed, hdr, gab=gab, epf_iters=epf_iters, ac_type=ac_type)
    else:
        desc, coeffs = wl.synthetic_frame(w, h, seed=seed, gab=gab, epf_iters=epf_iters, ac_type=ac_type)
    rng = np.random.default_rng(seed + 515)
    shape = desc.dc.shape[1:]
    kind = rng.integers(0, 3, shape)
    y = np.where(kind == 0, rng.uniform(1.5, 3.0, shape), np.where(kind == 1, rng.uniform(-0.6, -0.05, shape),
                                                                   rng.uniform(0.0, 1.5, shape)))
    desc.dc = desc.dc.copy()
    desc.dc[1] = y.astype(np.float32)
    if n > 1:
        desc.upsampling = n
        desc.upsampling_weights = (custom_upsampling_weights(n, seed) if weights == "custom"
                                   else default_upsampling_weights(n))
        desc.xsize_upsampled, desc.ysize_upsampled = n * w - (n - 1), n * h - 1
    if noise:
        desc.noise, desc.noise_lut = 1, tuple(lut)
        desc.visible_frame_index, desc.nonvisible_frame_index = frame_index
    desc.out_format, desc.stage_mask = fmt, srgb
    return desc, coeffs


def ups_decoy(desc: abi.FrameDesc, seed: int):
    """A frame of the same geometry, chain and output as the upsampled / noisy `desc` with other content, other
    frame indices (other noise) and other weights.  Rendered on a context just before `desc` it leaves ups_in,
    noise_raw, noise_buf and the tap table full of values that are wrong for `desc`."""
    import dataclasses
    d, coeffs = decoy_frame(desc, seed)
    n = desc.upsampling if desc.upsampling > 1 else 1
    # the frame's X, Y and B DC mirrored: where the frame saturates an 8-bit channel, the decoy does not
    dc = np.stack([-desc.dc[0], np.float32(1.4) - desc.dc[1], np.float32(0.6) - desc.dc[2]]).astype(np.float32)
    d = dataclasses.replace(d, dc=dc, visible_frame_index=desc.visible_frame_index + 7,
                            nonvisible_frame_index=desc.nonvisible_frame_index + 11)
    if n > 1:
        d.upsampling_weights = custom_upsampling_weights(n, seed + 1)
    return d, coeffs


def mirror_index(i: np.ndarray, size: int) -> np.ndarray:
    """Mirror() of image_ops.h: reflect (edge repeated) until inside [0, size)."""
    i = np.asarray(i, np.int64).copy()
    while True:
        lo, hi = i < 0, i >= size
        if not (lo.any() or hi.any()):
            return i
        i = np.where(lo, -i - 1, np.where(hi, 2 * size - 1 - i, i))


def tap_table(weights, n: int, transpose: bool = False) -> np.ndarray:
    """(n, n, 5, 5) float64 taps of output sub-pixel (ky, kx), built from the n/2 x n/2 x 25 weights as the symmetric
    (5n/2)^2 matrix whose upper triangle they list row by row: sub-pixels in the lower / right half use the mirrored
    sub-pixel and the mirrored window.  transpose: each 5x5 transposed (a deliberately wrong model)."""
    h = n // 2
    m = 5 * h
    w = np.asarray(weights, np.float64)
    assert w.size == m * (m + 1) // 2
    M = np.zeros((m, m))
    iu = np.triu_indices(m)
    M[iu] = w
    M[iu[1], iu[0]] = w
    t = np.zeros((n, n, 5, 5))
    for ky in range(n):
        for kx in range(n):
            fy, fx = ky if ky < h else n - 1 - ky, kx if kx < h else n - 1 - kx
            for py in range(5):
                for px in range(5):
                    j = 5 * fy + (py if ky < h else 4 - py)
                    i = 5 * fx + (px if kx < h else 4 - px)
                    t[ky, kx, py, px] = M[j, i]
    return t.transpose(0, 1, 3, 2).copy() if transpose else t


def upsample_model(planes: np.ndarray, weights, n: int, ow: int, oh: int, clamp: bool = True,
                   transpose: bool = False):
    """float64 UpsamplingStage: (3, h, w) planes -> (out, unclamped, sum|v*k|), each (3, oh, ow).  Input mirrored about
    the coded size; every output clamped to the min / max of its 5x5 input window."""
    c, h, w = planes.shape
    p = planes.astype(np.float64)
    ys, xs = mirror_index(np.arange(-2, h + 2), h), mirror_index(np.arange(-2, w + 2), w)
    pad = p[:, ys][:, :, xs]
    win = np.lib.stride_tricks.sliding_window_view(pad, (5, 5), axis=(1, 2))     # (3, h, w, 5, 5)
    mn, mx = win.min(axis=(3, 4)), win.max(axis=(3, 4))
    taps = tap_table(weights, n, transpose)
    raw = np.zeros((c, h * n, w * n))
    acc = np.zeros_like(raw)
    out = np.zeros_like(raw)
    for ky in range(n):
        for kx in range(n):
            k = taps[ky, kx]
            r = np.einsum("chwij,ij->chw", win, k)
            raw[:, ky::n, kx::n] = r
            acc[:, ky::n, kx::n] = np.einsum("chwij,ij->chw", np.abs(win), np.abs(k))
            out[:, ky::n, kx::n] = np.clip(r, mn, mx) if clamp else r
    return out[:, :oh, :ow], raw[:, :oh, :ow], acc[:, :oh, :ow]


def convolve_noise_model(raw: np.ndarray, mirror_wh=None):
    """float64 ConvolveNoiseStage of (3, H, W) generator planes: 0.16 * (sum of the 24 neighbours) - 3.84 * centre,
    borders mirrored about the output size (`mirror_wh`: about another size, a deliberately wrong model).
    Returns (conv, 0.16 * others + 3.84 * |centre| for the error bound)."""
    _, H, W = raw.shape
    mw, mh = mirror_wh or (W, H)
    r = raw.astype(np.float64)
    xs = [mirror_index(np.arange(W) + d, mw) for d in range(-2, 3)]
    ys = [mirror_index(np.arange(H) + d, mh) for d in range(-2, 3)]
    others = np.zeros_like(r)
    for dy in range(5):
        for dx in range(5):
            if dy != 2 or dx != 2:
                others += r[:, ys[dy]][:, :, xs[dx]]
    centre = r[:, ys[2]][:, :, xs[2]]
    return 0.16 * others - 3.84 * centre, 0.16 * others + 3.84 * np.abs(centre)


def noise_strength_model(lut, x: np.ndarray) -> np.ndarray:
    """StrengthEvalLut in float64."""
    lut = np.asarray(lut, np.float64)
    s = np.maximum(x * 6.0, 0.0)
    fl = np.floor(s)
    frac = s - fl
    sat = s >= 7.0
    fl, frac = np.where(sat, 6.0, fl), np.where(sat, 1.0, frac)
    i = fl.astype(np.int64)
    return np.clip(lut[i] + (lut[i + 1] - lut[i]) * frac, 0.0, 1.0)


def lut_segments(x: np.ndarray) -> np.ndarray:
    """Which branch of StrengthEvalLut an input takes: -1 negative (clamped to 0), 0..6 the segment, 7 saturated."""
    s = x * 6.0
    return np.where(s < 0, -1, np.where(s >= 7.0, 7, np.floor(np.maximum(s, 0)))).astype(np.int64)


def add_noise_model(xyb: np.ndarray, conv: np.ndarray, lut, cfl_x: float, cfl_b: float) -> np.ndarray:
    """float64 AddNoiseStage on (3, H, W) X, Y, B with the convolved noise planes."""
    X, Y, B = xyb
    rr, rg, rc = conv * 0.22
    sg, sr = noise_strength_model(lut, (Y - X) * 0.5), noise_strength_model(lut, (Y + X) * 0.5)
    red = sr * (0.0078125 * rr + 0.9921875 * rc)
    green = sg * (0.0078125 * rg + 0.9921875 * rc)
    s = red + green
    return np.stack([cfl_x * s + (red - green) + X, Y + s, cfl_b * s + B])


def ups_noise_coverage(desc: abi.FrameDesc, coeffs: np.ndarray, what: str = "", pre: np.ndarray | None = None,
                       min_segment: int = 100) -> dict:
    """What the frame exercises, in float64 from the oracle's pre-upsampling planes (`pre`: those planes if at hand):
    the fraction of output samples per channel that the window clamp changed (at least 1 %, and some in the ragged
    last 256-tile of every tile row and tile column), the number of AddNoise inputs (Y - X and Y + X) per branch of
    StrengthEvalLut (every one at least `min_segment`) and the output's raggedness.  Prints and returns the figures."""
    from oracle import cpu as ocpu
    if pre is None:
        pre = ocpu.render_frame(pre_upsampling_desc(desc), coeffs, rcp_mode=0)
    n = desc.upsampling if desc.upsampling > 1 else 1
    ow, oh = out_size(desc)
    res = {"out": (ow, oh)}
    assert ow % 256 and oh % 256, ("no ragged 256-tile", ow, oh)
    if n > 1:
        xyb, raw, _ = upsample_model(pre, desc.upsampling_weights, n, ow, oh)
        changed = xyb != raw
        res["clamp_frac"] = [float(changed[c].mean()) for c in range(3)]
        tx, ty = (ow // 256) * 256, (oh // 256) * 256
        right = [bool(changed[:, y0:y0 + 256, tx:].any()) for y0 in range(0, oh, 256)]
        bottom = [bool(changed[:, ty:, x0:x0 + 256].any()) for x0 in range(0, ow, 256)]
        assert min(res["clamp_frac"]) >= 0.01, (what, res["clamp_frac"])
        assert all(right) and all(bottom), (what, right, bottom)
    else:
        xyb = pre.astype(np.float64)
    if desc.noise:
        seg = np.concatenate([lut_segments((xyb[1] - xyb[0]) * 0.5).ravel(),
                              lut_segments((xyb[1] + xyb[0]) * 0.5).ravel()])
        counts = np.bincount(seg + 1, minlength=9)
        res["lut_counts"] = {"neg": int(counts[0]), **{str(i): int(counts[i + 1]) for i in range(7)},
                             "sat": int(counts[8])}
        assert counts.min() >= min_segment, (what, res["lut_counts"])
    print(f"coverage {what}: {n}x, output {ow}x{oh} (w % 16 = {ow % 16}, last tile {ow % 256}x{oh % 256}); "
          f"clamp fraction per channel {[f'{v:.2%}' for v in res.get('clamp_frac', [])]}; "
          f"LUT branches {res.get('lut_counts')}")
    return res


GAMMA_25 = 25 * 2.0 ** -24 / (1 - 25 * 2.0 ** -24)   # Higham's gamma_n: n float32 roundings in a row


def check_float64_model(p, desc: abi.FrameDesc, coeffs: np.ndarray, what: str = "") -> dict:
    """Render `desc` on the pipeline `p` as planar XYB (no colour stage) and compare it with the float64 models of
    the upsampling (from the n/2 triangular weights, not the kernel's table), ConvolveNoise and AddNoise, fed with
    the kernels' own pre-upsampling planes (a render of pre_upsampling_desc) and the oracle's generator planes.  The
    bound is counted per sample from the float32 operations (u = 2^-24 per rounding).  Asserts that the largest
    error is within it and, for upsampled frames, that three wrong models (5x5 taps transposed, no window clamp,
    noise mirrored about the coded size) exceed it at least 100 times.  Prints and returns the ratios."""
    import dataclasses
    from oracle import cpu as ocpu
    pre = p.decode_frame(pre_upsampling_desc(desc), coeffs)
    d = dataclasses.replace(desc, stage_mask=abi.STAGE_EXPLICIT | filter_mask(desc), out_format=abi.OUT_PLANAR_F32)
    got = p.decode_frame(d, coeffs).astype(np.float64)
    n = desc.upsampling if desc.upsampling > 1 else 1
    ow, oh = out_size(desc)
    u = 2.0 ** -24
    gen = ocpu.noise_planes(desc.visible_frame_index, desc.nonvisible_frame_index, ow, oh) if desc.noise else None
    lut = np.asarray(desc.noise_lut, np.float64)
    slope = 3.0 * np.abs(np.diff(lut)).max()      # d strength / d input (x * 0.5 * 6)

    def model(transpose=False, clamp=True, mirror=None):
        if n > 1:
            up, _, acc = upsample_model(pre, desc.upsampling_weights, n, ow, oh, clamp, transpose)
        else:
            up, acc = pre.astype(np.float64), np.zeros((3, oh, ow))
        e_up = GAMMA_25 * acc + u * np.abs(up)      # 25 products summed in any order, then the clamp
        if not desc.noise:
            return up, e_up + u * np.abs(up)
        conv, cmag = convolve_noise_model(gen, mirror)
        out = add_noise_model(up, conv, lut, desc.cfl_base_x, desc.cfl_base_b)
        X, Y, _ = up
        rnd = 0.22 * conv
        e_rnd = 0.22 * 30 * u * cmag + u * np.abs(rnd)
        m_r = 0.0078125 * rnd[0] + 0.9921875 * rnd[2]
        m_g = 0.0078125 * rnd[1] + 0.9921875 * rnd[2]
        e_mr = 0.0078125 * e_rnd[0] + 0.9921875 * e_rnd[2] + 2 * u * (np.abs(rnd[0]) + np.abs(rnd[2]))
        e_mg = 0.0078125 * e_rnd[1] + 0.9921875 * e_rnd[2] + 2 * u * (np.abs(rnd[1]) + np.abs(rnd[2]))
        e_s = slope * (e_up[0] + e_up[1] + 3 * u * (np.abs(X) + np.abs(Y))) + 4 * u
        sr = noise_strength_model(lut, (Y + X) * 0.5)
        sg = noise_strength_model(lut, (Y - X) * 0.5)
        red, green = sr * m_r, sg * m_g
        e_red = e_s * np.abs(m_r) + sr * e_mr + u * np.abs(red)
        e_green = e_s * np.abs(m_g) + sg * e_mg + u * np.abs(green)
        s = red + green
        e_sum = e_red + e_green + u * np.abs(s)
        cx, cb = abs(desc.cfl_base_x), abs(desc.cfl_base_b)
        bound = np.stack([
            e_up[0] + cx * e_sum + e_red + e_green + 3 * u * (cx * np.abs(s) + np.abs(red) + np.abs(green) + np.abs(out[0])),
            e_up[1] + e_sum + u * np.abs(out[1]),
            e_up[2] + cb * e_sum + 2 * u * (cb * np.abs(s) + np.abs(out[2]))])
        return out, bound

    want, bound = model()
    ratio = float((np.abs(got - want) / bound).max())
    res = {"ratio": ratio}
    if n > 1:
        wrong = {"transposed taps": model(transpose=True)[0], "no clamp": model(clamp=False)[0]}
        if desc.noise:
            wrong["noise mirrored about the coded size"] = model(mirror=(desc.xsize, desc.ysize))[0]
        res.update({k: float((np.abs(got - v) / bound).max()) for k, v in wrong.items()})
    print(f"float64 model {what}: largest error {ratio:.3g} of the bound; wrong models: "
          f"{ {k: f'{v:.3g}' for k, v in res.items() if k != 'ratio'} }")
    assert ratio <= 1.0, (what, ratio)
    assert all(v >= 100 for k, v in res.items() if k != "ratio"), (what, res)
    return res


def dc_stage_input(xs: int, ys: int) -> np.ndarray:
    """Seeded quantised DC planes (X, Y, B): smooth gradients (adaptive smoothing engages) with one busy
    quadrant (it must switch itself off there)."""
    rng = np.random.default_rng(1000 * xs + ys)
    yy, xx = np.mgrid[0:ys, 0:xs]
    q = np.stack([np.round(20 * np.sin(xx / 17 + c) + 15 * np.cos(yy / 23 + c) + rng.random((ys, xs)) * 1.2)
                  for c in range(3)]).astype(np.int32)
    q[:, ys // 2:, xs // 2:] += rng.integers(-40, 40, (3, ys - ys // 2, xs - xs // 2))
    return q
