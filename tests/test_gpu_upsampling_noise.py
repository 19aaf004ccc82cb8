"""-m gpu: upsampling (2x / 4x / 8x) and noise where they engage.  Custom F16 weights, a strength LUT that reaches
every branch of StrengthEvalLut, ragged output sizes (support.ups_noise_frame), every output format, filter chain and
entry point; each checked render follows a decoy of other content, frame indices and weights, so a kernel that skips
a region cannot pass on what the previous render left in ups_in, noise_raw, noise_buf or the tap table.  Bit-exact
against the oracle (rcp_mode 0).  The emulator mirror is tests/test_emulated_upsampling_noise.py."""
import time

import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi, pipeline
from tests import support

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("built")]

FORMATS = [(abi.OUT_RGB_F32, 0), (abi.OUT_PLANAR_F32, 0), (abi.OUT_RGB_U8, abi.STAGE_SRGB),
           (abi.OUT_RGBA_U8, abi.STAGE_SRGB), (abi.OUT_RGB_U16, 0), (abi.OUT_RGB_F16, abi.STAGE_SRGB)]
# coded sizes; outputs 1201 x 565, 1197 x 1079, 1193 x 799: ragged 256-tiles, widths not multiples of 16
SIZES = {2: (601, 283), 4: (300, 270), 8: (150, 100)}


@pytest.fixture(scope="module", params=["two-kernel", "fused"])
def pipe(request):
    """Both module contexts; the fused one falls back to the two-kernel path for these frames."""
    import os
    old = os.environ.get("JXLGPU_FUSED")
    os.environ["JXLGPU_FUSED"] = "1" if request.param == "fused" else "0"
    try:
        p = pipeline.TransformPipeline(device=0, num_host_threads=4)
        yield p
        p.close()
    finally:
        if old is None:
            os.environ.pop("JXLGPU_FUSED", None)
        else:
            os.environ["JXLGPU_FUSED"] = old


def oracle(desc, coeffs):
    from oracle import cpu
    return cpu.render_frame(desc, coeffs, rcp_mode=0)


def assert_same(got, want, what=""):
    from tests.test_gpu_parity import assert_same as same
    same(got, want, what)


def after_decoy(p, desc, coeffs, seed, render=None, want=None, decoy_of=None):
    """Render a decoy (support.ups_decoy of `decoy_of`, default the frame) on `p`, then the frame; the decoy must
    differ from the frame on 99 % of the pixels.  Returns (frame's render, oracle)."""
    render = render or (lambda d, c: p.decode_frame(d, c))
    want = oracle(desc, coeffs) if want is None else want
    d, dc = support.ups_decoy(desc if decoy_of is None else decoy_of, seed)
    decoy = render(d, dc)
    assert_same(decoy, oracle(d, dc), "decoy")
    # (8-bit outputs: pixels that both saturate to the same corner of the cube coincide, up to 1.5 % of them)
    eight = desc.out_format in (abi.OUT_RGB_U8, abi.OUT_RGBA_U8)
    support.assert_decoy_differs(decoy, want, desc.out_format == abi.OUT_PLANAR_F32, 0.98 if eight else 0.99)
    return render(desc, coeffs), want


@pytest.mark.parametrize("n", [1, 2, 4, 8])
def test_scenario_coverage(n):
    """What the frames of this file reach: window clamp fraction, AddNoise inputs per LUT branch, ragged tiles."""
    w, h = SIZES.get(n, (1201, 531))
    desc, coeffs = support.ups_noise_frame(n, w, h, seed=10 * n)
    support.ups_noise_coverage(desc, coeffs, f"{n}x {w}x{h}")


@pytest.mark.parametrize("fmt,srgb", FORMATS)
@pytest.mark.parametrize("noise", [0, 1])
@pytest.mark.parametrize("n", [2, 4, 8])
def test_factor_noise_format(pipe, n, noise, fmt, srgb):
    w, h = SIZES[n]
    desc, coeffs = support.ups_noise_frame(n, w, h, seed=10 * n, noise=bool(noise), fmt=fmt, srgb=srgb)
    got, want = after_decoy(pipe, desc, coeffs, seed=500 + fmt)
    assert_same(got, want, f"{n}x noise={noise} fmt={fmt}")


@pytest.mark.parametrize("gab", [0, 1])
@pytest.mark.parametrize("epf_iters", [0, 1, 2, 3])
def test_production_chains(pipe, gab, epf_iters):
    """The eight chains PreparePipeline builds, at 4x with noise: the strip kernel runs them without its XYB stage."""
    desc, coeffs = support.ups_noise_frame(4, 300, 270, seed=gab * 4 + epf_iters, gab=gab, epf_iters=epf_iters)
    got, want = after_decoy(pipe, desc, coeffs, seed=gab + 10 * epf_iters)
    assert_same(got, want, f"gab={gab} epf={epf_iters}")


@pytest.mark.parametrize("mask", [None, abi.STAGE_GAB | abi.STAGE_EPF2 | abi.STAGE_XYB, abi.STAGE_EPF0 | abi.STAGE_XYB])
def test_generic_tile_kernel(mask, monkeypatch):
    """JXLGPU_FORCE_GENERIC_FILTER=1 (read when a context is created) on the production chain, and explicit chains
    outside the production set: the generic tile kernel writes ups_in."""
    if mask is None:
        monkeypatch.setenv("JXLGPU_FORCE_GENERIC_FILTER", "1")
    p = pipeline.TransformPipeline(device=0, num_host_threads=1)
    try:
        desc, coeffs = support.ups_noise_frame(4, 300, 270, seed=77, epf_iters=3)
        if mask is not None:
            desc.stage_mask = abi.STAGE_EXPLICIT | mask
        got, want = after_decoy(p, desc, coeffs, seed=78)
        assert_same(got, want, f"generic {mask}")
    finally:
        p.close()


@pytest.mark.parametrize("fmt,srgb", [(abi.OUT_RGB_F32, 0), (abi.OUT_RGB_U8, abi.STAGE_SRGB)])
def test_large_frame_8x_with_noise(fmt, srgb):
    """960 x 540 coded at 8x with noise: a 7673 x 4319 output (30 x 17 noise tiles, ragged in both directions), int32
    coefficients.  Whole-image compare; the oracle's time is printed."""
    p = pipeline.TransformPipeline(device=0, num_host_threads=4)
    try:
        desc, coeffs = support.ups_noise_frame(8, 960, 540, seed=960, fmt=fmt, srgb=srgb, ac_type=abi.AC_INT32)
        t0 = time.perf_counter()
        want = oracle(desc, coeffs)
        print(f"oracle: {time.perf_counter() - t0:.1f} s for {desc.out_shape()}")
        got, _ = after_decoy(p, desc, coeffs, seed=961, want=want)
        assert_same(got, want, "8x large")
    finally:
        p.close()


def test_render_device_padded_stride_on_a_torch_stream(pipe):
    """render_device on a caller's stream into rows longer than the pixels: padding untouched, and the launches are
    the noise generator + convolution at frame_begin, then the transforms, the filter and upsample_in_kernel."""
    import torch
    desc, coeffs = support.ups_noise_frame(4, 300, 270, seed=31)
    row = desc.out_row_bytes
    stride = row + 256
    oh = desc.out_shape()[0]
    dev = torch.from_numpy(coeffs).cuda()
    stream = torch.cuda.Stream()

    def render(d, c):
        dv = torch.from_numpy(c).cuda()
        buf = torch.full((oh, stride), 0x5A, dtype=torch.uint8, device="cuda")
        pipe.set_device_coefficients([dv[k].data_ptr() for k in range(3)])
        try:
            n0 = pipe.launch_count()
            pipe.frame_begin(d)
            n1 = pipe.launch_count()
            stream.wait_stream(torch.cuda.current_stream())     # (the fill above ran on the current stream)
            pipe.render_device(buf.data_ptr(), stride, stream.cuda_stream)
            stream.synchronize()
            n2 = pipe.launch_count()
        finally:
            pipe.set_device_coefficients(None)
        assert n1 - n0 == 2 and n2 - n1 == 7, (n1 - n0, n2 - n1)   # plan, mid, large rows + columns, idct8, filter, ups
        b = buf.cpu().numpy()
        assert (b[:, row:] == 0x5A).all()
        return b[:, :row].copy().view(np.float32).reshape(d.out_shape())

    got, want = after_decoy(pipe, desc, coeffs, seed=32, render=render)
    del dev
    assert_same(got, want, "render_device")


def test_host_fed_streaming_and_sparse(pipe):
    """Shuffled submission with stream_output into a pinned buffer, and the sparse hand-off (int16 and int32)."""
    desc, coeffs = support.ups_noise_frame(4, 600, 530, seed=41, fmt=abi.OUT_RGB_U8, srgb=abi.STAGE_SRGB)
    order = np.random.default_rng(1).permutation(desc.num_groups)

    def streamed(d, c):
        out = pipeline.pinned_array(d.out_shape(), d.out_dtype)
        out[:] = 7
        got = pipe.decode_frame(d, c, out=out, order=order, stream_output=True)
        assert got is out
        return got.copy()

    got, want = after_decoy(pipe, desc, coeffs, seed=42, render=streamed)
    assert_same(got, want, "streamed")
    got, _ = after_decoy(pipe, desc, coeffs, seed=43, want=want,
                         render=lambda d, c: pipe.decode_frame(d, c, sparse=True, order=order.tolist()))
    assert_same(got, want, "sparse int16")
    desc, coeffs = support.ups_noise_frame(8, 200, 150, seed=44, ac_type=abi.AC_INT32)
    coeffs = coeffs.copy()
    rng = np.random.default_rng(2)
    for c in range(3):
        g, k = rng.integers(0, desc.num_groups, 50), rng.integers(64, 4096, 50)
        coeffs[c, g, k] = rng.integers(-300000, 300000, 50)
    got, want = after_decoy(pipe, desc, coeffs, seed=45, render=lambda d, c: pipe.decode_frame(d, c, sparse=True))
    assert_same(got, want, "sparse int32")


def test_dc_stage_on_the_device(pipe):
    """Quantised DC in, DequantDC + AdaptiveDCSmoothing on the device, then the upsampling and the noise (after a
    decoy with host-prepared DC)."""
    import dataclasses
    from tests.test_zz_dc_stage_gpu import with_quant_dc
    desc, coeffs = support.ups_noise_frame(4, 520, 264, seed=51)
    q, gm, dc = with_quant_dc(desc, 1)
    desc.dc = dc
    want = oracle(desc, coeffs)
    host_dc = dataclasses.replace(desc)
    desc.quant_dc, desc.dc_group_mul, desc.dc_smoothing = q, gm, 1
    desc.dc_factors, desc.dc_cfl_factors = support.DC_FACTORS, support.DC_CFL
    desc.dc = None
    assert_same(oracle(desc, coeffs), want, "oracle: DC stage")
    got, _ = after_decoy(pipe, desc, coeffs, seed=52, want=want, decoy_of=host_dc)
    assert_same(got, want, "DC stage")


@pytest.mark.parametrize("hdr", list(wl.HEADER_SETS) + [12])
@pytest.mark.parametrize("n", [4, 8])
def test_header_sets(pipe, n, hdr):
    w, h = SIZES[n]
    desc, coeffs = support.ups_noise_frame(n, w, h, seed=60 + n, hdr=hdr, epf_iters=3)
    got, want = after_decoy(pipe, desc, coeffs, seed=61)
    assert_same(got, want, f"{n}x {hdr}")


def test_context_sequence():
    """One context: frames whose upsampling / noise state (tap table, noise planes, host output, buffer sizes) must be
    reset or re-sized between them, each against the oracle."""
    p = pipeline.TransformPipeline(device=0, num_host_threads=2)
    try:
        seq = [support.ups_noise_frame(8, 960, 540, seed=1),
               support.ups_noise_frame(2, 601, 283, seed=2, noise=False),
               wl.synthetic_frame(700, 500, seed=3, epf_iters=1),
               support.ups_noise_frame(1, 1201, 531, seed=4, frame_index=(9, 2)),
               support.ups_noise_frame(4, 300, 270, seed=5),
               support.ups_noise_frame(8, 41, 23, seed=6)]
        for i, (desc, coeffs) in enumerate(seq):
            assert_same(p.decode_frame(desc, coeffs), oracle(desc, coeffs), f"frame {i}")
    finally:
        p.close()


@pytest.mark.parametrize("n", [1, 4, 8])
def test_float64_model(pipe, n):
    """The planar XYB output against support.check_float64_model: the upsampling from the triangular weights,
    ConvolveNoise and AddNoise in float64, on the kernels' own pre-upsampling planes; three wrong models exceed the
    bound by at least 100 times."""
    w, h = SIZES.get(n, (1201, 531))
    desc, coeffs = support.ups_noise_frame(n, w, h, seed=70 + n)
    support.check_float64_model(pipe, desc, coeffs, f"{n}x")


@pytest.mark.parametrize("rs,w,h", [(4, 1101, 517), (8, 2101, 167)])
def test_photon_noise_reference_frames(pipe, rs, w, h):
    """Codestreams the reference encoder makes (oracle/_ref) with resampling 4 / 8 and photon noise: entropy-decoded
    by the reference, rendered here after a decoy, bit-exact against the oracle and within the tolerance of
    test_upsampled_reference_frames of the reference decoder's own pixels."""
    from oracle import cpu, ref
    if not ref.available():
        pytest.skip("oracle/_ref not built")
    data = ref.encode_rgb8(wl.synth_image(w, h, seed=rs + 3200), 1.0, 7, -1, -1, 4, resampling=rs | (32 << 16))
    fr = ref.Frame(data, 2)
    d = fr.dump()
    fr.close()
    desc = cpu.desc_from_dump(d)
    assert desc.upsampling == rs and desc.noise == 1 and desc.out_shape() == (h, w, 3)
    got, want = after_decoy(pipe, desc, d.coeffs, seed=rs)
    assert_same(got, want, f"resampling {rs} + noise vs oracle")
    assert np.abs(got - d.decoded).max() <= 2e-5       # vs the reference decoder (rcpps in AdjustQuantBias)


@pytest.mark.parametrize("mode", ["ce", "sm", "kernel"])
def test_replicas_refused(mode, monkeypatch):
    """Output replicas (three more buffers on this device) with an upsampled and a noisy frame: render_device refuses
    them (JXLGPU_ERR_UNSUPPORTED) without writing anything, and the context renders the next frame."""
    import torch
    if mode == "ce":
        monkeypatch.delenv("JXLGPU_GATHER", raising=False)
    else:
        monkeypatch.setenv("JXLGPU_GATHER", mode)
    p = pipeline.TransformPipeline(device=0, num_host_threads=1)
    try:
        for desc, coeffs in (support.ups_noise_frame(4, 300, 270, seed=80, noise=False),
                             support.ups_noise_frame(1, 1201, 531, seed=81)):
            dev = torch.from_numpy(coeffs).cuda()
            bufs = [torch.full(desc.out_shape(), 3.0, dtype=torch.float32, device="cuda") for _ in range(4)]
            p.set_device_coefficients([dev[c].data_ptr() for c in range(3)])
            p.frame_begin(desc)
            p.set_output_replicas([b.data_ptr() for b in bufs[1:]])
            before = p.launch_count()
            try:
                with pytest.raises(pipeline.JxlGpuError) as e:
                    p.render_device(bufs[0].data_ptr(), desc.out_row_bytes, torch.cuda.current_stream().cuda_stream)
                assert e.value.code == abi.ERR_UNSUPPORTED
            finally:
                p.set_output_replicas([])
                p.set_device_coefficients(None)
            torch.cuda.synchronize()
            assert p.launch_count() == before
            assert all(bool((b == 3.0).all()) for b in bufs)
            assert_same(p.decode_frame(desc, coeffs), oracle(desc, coeffs), "after the refusal")
    finally:
        p.close()
