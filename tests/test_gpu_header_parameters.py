"""-m gpu: the kernels at non-default frame-header / image-metadata parameters.

About 25 scalars of jxlgpu_frame come from the frame header and the image metadata: the Gaborish weights, the EPF
sharpness LUT, channel scales, sigma scales and border multiplier, the CfL base correlations and colour factor, the
quantisation biases, the X / B dequantisation multipliers and the inverse opsin matrix and biases.  The default
values hide whole classes of bugs (the same Gaborish weights and opsin biases for X, Y and B, a CfL base of 0 / 1,
a sharpness LUT of i / 7, an intensity target of 255), so every test here runs the legal non-default header sets
of jxl_workload.header_params:
  * every device path at a non-default set, bit-exact against the oracle (exact-reciprocal mode);
  * a one-at-a-time sensitivity sweep over every scalar (each channel separately): the oracle's output moves,
    and the GPU follows it bit for bit;
  * frames the reference encoder made, with the header overridden in the reference's own frame state
    (oracle.ref.Frame.set_params): the GPU against the reference's stage output;
  * a float64 model of Gaborish and XYB -> linear, independent of the oracle and of libjxl, applied to the
    GPU's own stage taps."""
import os

import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi, pipeline
from tests import support
from tests.test_gpu_parity import assert_same

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("built")]

CONTEXTS = {"two-kernel": {"JXLGPU_FUSED": "0"}, "fused": {"JXLGPU_FUSED": "1"},
            "idct8": {"JXLGPU_FUSED": "0", "JXLGPU_IDCT8_TMA": "0"}}


@pytest.fixture(scope="module")
def pipes():
    """One context per device path that is chosen when the context is created (environment read then)."""
    made = {}

    def get(name):
        if name not in made:
            saved = {k: os.environ.get(k) for k in ("JXLGPU_FUSED", "JXLGPU_IDCT8_TMA")}
            os.environ.update(CONTEXTS[name])
            try:
                made[name] = pipeline.TransformPipeline(device=0, num_host_threads=4)
            finally:
                for k, v in saved.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
        return made[name]
    yield get
    for p in made.values():
        p.close()


def oracle(desc, coeffs):
    from oracle import cpu
    return cpu.render_frame(desc, coeffs, rcp_mode=0)


FORMATS = {"f32": (abi.OUT_RGB_F32, 0), "srgb8": (abi.OUT_RGB_U8, abi.STAGE_SRGB)}
# the eight chains PreparePipeline builds -> strip-kernel masks 16, 17, 20, 21, 28, 29, 30, 31
CHAINS = [(gab, epf) for epf in range(4) for gab in range(2)]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("gab,epf_iters", CHAINS)
def test_strip_kernel_chains(pipes, gab, epf_iters, fmt):
    hdr = wl.HEADER_SETS[(2 * epf_iters + gab) % 3]
    ac = abi.AC_INT32 if epf_iters % 2 else abi.AC_INT16
    desc, coeffs = support.header_frame(531, 300, seed=10 + 2 * epf_iters + gab, hdr=hdr, gab=gab,
                                        epf_iters=epf_iters, ac_type=ac)
    desc.out_format, desc.stage_mask = FORMATS[fmt]
    assert_same(pipes("two-kernel").decode_frame(desc, coeffs), oracle(desc, coeffs), f"{hdr} gab={gab} epf={epf_iters}")


# (path, context, header set, coefficient type)
PATHS = [("tile", "two-kernel", "dim80", abi.AC_INT16), ("fused", "fused", "pq10000", abi.AC_INT32),
         ("idct8", "idct8", "edges", abi.AC_INT16), ("upsampling2", "two-kernel", "pq10000", abi.AC_INT32),
         ("noise", "two-kernel", "edges", abi.AC_INT16), ("noise_upsampling2", "two-kernel", "dim80", abi.AC_INT32),
         ("ycbcr", "two-kernel", 17, abi.AC_INT16), ("dc_stage", "two-kernel", "dim80", abi.AC_INT32),
         ("sparse", "two-kernel", 23, abi.AC_INT32), ("sparse_fused", "fused", "edges", abi.AC_INT16)]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("path,ctx,hdr,ac", PATHS, ids=[p[0] for p in PATHS])
def test_device_paths(pipes, path, ctx, hdr, ac, fmt):
    from tests.test_emulated_cuda import NOISE_LUT
    w, h = (301, 211) if "upsampling" in path else (777, 523)
    desc, coeffs = support.header_frame(w, h, seed=len(path) * 31 + ac, hdr=hdr, gab=1,
                                        epf_iters=1 if "upsampling" in path else 2, ac_type=ac)
    desc.out_format, desc.stage_mask = FORMATS[fmt]
    if path == "tile":        # an explicit chain outside the production set
        desc.stage_mask |= abi.STAGE_EXPLICIT | abi.STAGE_GAB | abi.STAGE_EPF2 | abi.STAGE_XYB
    if "upsampling" in path:
        wts = np.load(support.GOLDEN / "upsampling_weights.npz")
        desc.upsampling, desc.upsampling_weights = 2, wts["weights2"]
        desc.xsize_upsampled, desc.ysize_upsampled = 2 * w - 1, 2 * h - 1
    if path.startswith("noise"):
        desc.noise, desc.noise_lut = 1, NOISE_LUT
        desc.visible_frame_index, desc.nonvisible_frame_index = 2, 1
    if path == "ycbcr":
        desc.color_transform = 1
    if path == "dc_stage":
        from tests.test_zz_dc_stage_gpu import with_quant_dc
        q, gm, _ = with_quant_dc(desc, 1)
        desc.quant_dc, desc.dc_group_mul, desc.dc_smoothing = q, gm, 1
        desc.dc_factors, desc.dc_cfl_factors = support.DC_FACTORS, support.DC_CFL
        desc.dc = None
    want = oracle(desc, coeffs)
    got = pipes(ctx).decode_frame(desc, coeffs, sparse=path.startswith("sparse"))
    assert_same(got, want, f"{path} at header {hdr}")


def sweep_frame(noise: bool):
    """EPF engaged with all three passes after Gaborish (strip-kernel chain 31), every sharpness value present,
    at a non-default base header; with `noise`, the noise stages read the CfL base correlations too."""
    from tests.test_emulated_cuda import NOISE_LUT
    desc, coeffs = support.header_frame(300, 264, seed=91, hdr="dim80")
    desc.out_format = abi.OUT_PLANAR_F32
    if noise:
        desc.noise, desc.noise_lut = 1, NOISE_LUT
        desc.visible_frame_index, desc.nonvisible_frame_index = 1, 0
    return desc, coeffs


@pytest.mark.parametrize("noise", [False, True], ids=["filters", "noise"])
def test_one_at_a_time_sensitivity(pipes, noise):
    """Each scalar of support.SWEEP_FIELDS (each channel separately) is moved on its own from the base header:
    the oracle's output must change (the frame exercises the parameter) and the GPU must equal the oracle."""
    desc, coeffs = sweep_frame(noise)
    pipe = pipes("two-kernel")
    base = oracle(desc, coeffs)
    assert_same(pipe.decode_frame(desc, coeffs), base, "base header")
    entries = support.sweep_entries(support.NOISE_SWEEP if noise else support.SWEEP_FIELDS)
    inert = []
    for field, idx in entries:
        d = support.perturbed(desc, field, idx)
        want = oracle(d, coeffs)
        if np.array_equal(want, base):
            inert.append((field, idx))
        assert_same(pipe.decode_frame(d, coeffs), want, f"{field}[{idx}]")
    assert not inert, f"the sweep frame does not exercise {inert}"


@pytest.mark.parametrize("hdr,cfg", [("dim80", dict(w=517, h=331, distance=1.0, gaborish=1, epf=3)),
                                     ("pq10000", dict(w=640, h=264, distance=3.0, gaborish=1, epf=2)),
                                     ("edges", dict(w=600, h=300, distance=0.5, gaborish=1, epf=1))])
def test_reference_frames_with_overridden_header(pipes, hdr, cfg):
    """A codestream of the reference encoder, opened by the reference's FrameDecoder, with a non-default header
    written into its frame state: the GPU against the reference's own stages (the 12-bit rcpps of its
    AdjustQuantBias allows 2e-5 on the XYB planes, one code value in 8-bit sRGB) and bit-exact against the
    oracle.  (Linear f32 is compared with the oracle only: the rcpps error reaches linear light through
    3 g^2 times the opsin matrix, which these headers raise several-fold.)"""
    from oracle import cpu, ref
    if not (ref.available() and ref.available("strict")):
        pytest.skip("oracle/_ref not built")
    ref.use_variant("strict")
    try:
        if not ref.can_set_params():
            pytest.skip("oracle/_ref was built from a harness without ref_frame_set_params")
        data = ref.encode_rgb8(wl.synth_image(cfg["w"], cfg["h"], 41), cfg["distance"], 7, cfg["gaborish"], cfg["epf"], 2)
        fr = ref.Frame(data, 2)
        fr.set_params(wl.header_params(hdr))
        d = fr.dump()
        i = d.info
        chain = (1 if i.gab else 0) | (2 if i.epf_iters >= 3 else 0) | (4 if i.epf_iters >= 1 else 0) | \
            (8 if i.epf_iters >= 2 else 0)
        want_xyb, _ = fr.render(chain)
        want_u8, _ = fr.render_out(-33, abi.OUT_RGB_U8)
        fr.close()
    finally:
        ref.use_variant("default")
    pipe = pipes("two-kernel")
    desc = cpu.desc_from_dump(d, out_format=abi.OUT_PLANAR_F32, stage_mask=abi.STAGE_EXPLICIT | chain)
    got = pipe.decode_frame(desc, d.coeffs)
    assert_same(got, oracle(desc, d.coeffs), f"{hdr}: XYB planes vs oracle")
    assert np.abs(got - want_xyb).max() <= 2e-5
    desc.out_format, desc.stage_mask = abi.OUT_RGB_F32, 0
    assert_same(pipe.decode_frame(desc, d.coeffs), oracle(desc, d.coeffs), f"{hdr}: linear f32 vs oracle")
    desc.out_format, desc.stage_mask = abi.OUT_RGB_U8, abi.STAGE_SRGB
    got8 = pipe.decode_frame(desc, d.coeffs)
    assert_same(got8, oracle(desc, d.coeffs), f"{hdr}: sRGB u8 vs oracle")
    diff = np.abs(got8.astype(np.int16) - want_u8.astype(np.int16))
    assert diff.max() <= 1 and (diff != 0).mean() < 2e-3


# ---------------------------------------------------------------------------------------------------------------
# float64 model of the two per-channel, per-pixel stages
# ---------------------------------------------------------------------------------------------------------------
U = 2.0 ** -24          # unit roundoff of float32


def gaborish64(x, weights):
    """Normalised 3x3 Gaborish per channel, the image mirrored about its edge (x[-1] = x[0]).
    Returns (out, S) with S = sum |w_k x_k| over the nine taps."""
    out, s = np.empty_like(x), np.empty_like(x)
    for c in range(3):
        w1, w2 = weights[2 * c], weights[2 * c + 1]
        div = 1.0 + 4.0 * (w1 + w2)
        wc, we, wd = 1.0 / div, w1 / div, w2 / div
        p = np.pad(x[c], 1, mode="symmetric")
        ctr = p[1:-1, 1:-1]
        edges = [p[:-2, 1:-1], p[2:, 1:-1], p[1:-1, :-2], p[1:-1, 2:]]
        corners = [p[:-2, :-2], p[:-2, 2:], p[2:, :-2], p[2:, 2:]]
        out[c] = wc * ctr + we * sum(edges) + wd * sum(corners)
        s[c] = abs(wc) * np.abs(ctr) + abs(we) * sum(np.abs(e) for e in edges) + abs(wd) * sum(np.abs(e) for e in corners)
    return out, s


def xyb_to_linear64(x, m, bias, cbrt_bias):
    """XYB -> linear: L = Y + X, M = Y - X, S = B, minus the cube roots of the biases, cubed, plus the biases,
    times the inverse opsin matrix.  Returns (out, first-order float32 error bound)."""
    m = np.asarray(m, np.float64).reshape(3, 3)
    g = np.stack([x[1] + x[0], x[1] - x[0], x[2]]) - np.asarray(cbrt_bias, np.float64)[:, None, None]
    # gamma: two roundings (sum, bias subtraction) relative to |X| + |Y| + |cbrt|
    e_g = 2 * U * (np.stack([np.abs(x[1]) + np.abs(x[0])] * 2 + [np.abs(x[2])])
                   + np.abs(np.asarray(cbrt_bias, np.float64))[:, None, None])
    mixed = g ** 3 + np.asarray(bias, np.float64)[:, None, None]
    # cube + bias: the propagated 3 g^2 e_g, up to two roundings of the cube, one of the bias addition
    e_m = 3 * g * g * e_g + 2 * U * np.abs(g) ** 3 + U * np.abs(mixed)
    out = np.einsum("ij,jyx->iyx", m, mixed)
    # matrix row: three products summed, at most three roundings on each term
    e = np.einsum("ij,jyx->iyx", np.abs(m), e_m) + 3 * U * np.einsum("ij,jyx->iyx", np.abs(m), np.abs(mixed))
    return out, e


@pytest.mark.parametrize("hdr", ["dim80", "edges", 29])
def test_float64_model_of_gaborish_and_xyb(pipes, hdr):
    """The GPU's own taps: STAGE_EXPLICIT mask 0 (XYB after the transforms) as input, mask 1 (Gaborish) and
    mask 16 (XYB -> linear) as outputs, against plain float64 numpy.  Tolerances from the float32 operation count:
      * Gaborish: each normalised weight carries up to 5 roundings (w1 + w2, 4 *, + 1, 1 / div, w * (1 / div)),
        its product 1, the nine-term sum up to 8: |err| <= gamma_14 * sum |w_k x_k|, gamma_n = n u / (1 - n u);
      * XYB -> linear: the first-order bound propagated through each operation (xyb_to_linear64), times 1.01 for
        the second-order terms."""
    desc, coeffs = support.header_frame(419, 277, seed=5, hdr=hdr, gab=1, epf_iters=0)
    desc.out_format = abi.OUT_PLANAR_F32
    pipe = pipes("two-kernel")

    def tap(mask):
        desc.stage_mask = abi.STAGE_EXPLICIT | mask
        return pipe.decode_frame(desc, coeffs).astype(np.float64)
    x0, x_gab, x_lin = tap(0), tap(abi.STAGE_GAB), tap(abi.STAGE_XYB)
    gam14 = 14 * U / (1 - 14 * U)
    want, s = gaborish64(x0, desc.gab_weights)
    err = np.abs(x_gab - want)
    assert (err <= gam14 * s).all(), f"Gaborish: max err / bound {float((err / np.maximum(gam14 * s, 1e-30)).max()):.3f}"
    want, bound = xyb_to_linear64(x0, desc.inverse_opsin_matrix, desc.opsin_biases, desc.opsin_biases_cbrt)
    err = np.abs(x_lin - want)
    assert (err <= 1.01 * bound).all(), f"XYB: max err / bound {float((err / np.maximum(bound, 1e-30)).max()):.3f}"
    # the model is not trivially satisfied: a channel-0-only variant of either stage is far outside the bounds
    wrong, _ = gaborish64(x0, tuple(desc.gab_weights[:2]) * 3)
    assert (np.abs(x_gab - wrong) > gam14 * s).any()
    wrong, _ = xyb_to_linear64(x0, desc.inverse_opsin_matrix, (desc.opsin_biases[0],) * 3, (desc.opsin_biases_cbrt[0],) * 3)
    assert (np.abs(x_lin - wrong) > 1.01 * bound).any()
