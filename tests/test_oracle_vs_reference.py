"""Pins oracle/jxl_oracle.c against the UNMODIFIED reference compiled here by
oracle/build_ref.py (skipped where oracle/_ref is absent, e.g. a box without /root/reference
and without the prebuilt .so).  strict build = -ffp-contract=off => bit-exact expected."""
import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi
from tests import support

pytestmark = pytest.mark.usefixtures("built")


@pytest.fixture(scope="module")
def refmod(ref_available):
    if not ref_available:
        import os
        if os.path.isdir(os.environ.get("JXL_REFERENCE_ROOT", "/root/reference")):
            pytest.fail("oracle/_ref is not built although the reference is present: the oracle (and the tables it "
                        "shares with the product, csrc/jxl_tables.h) would go unpinned -- run `python oracle/build_ref.py`")
        pytest.skip("oracle/_ref not built (no reference on this box)")
    from oracle import ref
    ref.use_variant("strict")
    yield ref
    ref.use_variant("default")


def set_header(refmod, fr, hdr):
    """Frame.set_params with a non-default header set (jxl_workload.header_params); a harness prebuilt without
    ref_frame_set_params is a skip only where the reference sources are not there to rebuild it."""
    import os
    if not refmod.can_set_params():
        if os.path.isdir(os.environ.get("JXL_REFERENCE_ROOT", "/root/reference")):
            pytest.fail("oracle/_ref predates ref_frame_set_params although the reference is present: "
                        "run `python oracle/build_ref.py`")
        pytest.skip("oracle/_ref was built from a harness without ref_frame_set_params")
    fr.set_params(wl.header_params(hdr))


@pytest.mark.parametrize("strategy", range(27))
def test_all_strategies_bit_exact(strategy, refmod):
    from oracle import cpu
    rng = np.random.default_rng(1000 + strategy)
    r, c = abi.COVERED_Y[strategy] * 8, abi.COVERED_X[strategy] * 8
    for trial in range(2):
        co = (rng.laplace(0, 1.0, r * c) * (rng.random(r * c) < 0.3)).astype(np.float32)
        assert np.array_equal(refmod.transform_to_pixels(strategy, co, r, c), cpu.transform_to_pixels(strategy, co))
    dc = rng.normal(0, 1, (abi.COVERED_Y[strategy], abi.COVERED_X[strategy])).astype(np.float32)
    z = np.zeros(r * c, np.float32)
    assert np.array_equal(refmod.llf_from_dc(strategy, dc, z), cpu.llf_from_dc(strategy, dc, z))


@pytest.mark.parametrize("cfg", [
    dict(w=517, h=331, distance=1.0, gaborish=1, epf=3),      # odd size, full chain
    dict(w=512, h=512, distance=1.0, gaborish=-1, epf=-1),    # BASELINE config 1 (defaults: gab, epf 1)
    dict(w=300, h=520, distance=0.5, gaborish=0, epf=0),      # no filters: dequant+IDCT+XYB only
    dict(w=640, h=264, distance=3.0, gaborish=1, epf=2, kind="smooth"),  # large transforms
    # the same kinds of frame with a full non-default header written into the reference's frame state
    dict(w=517, h=331, distance=1.0, gaborish=1, epf=3, hdr="dim80"),
    dict(w=640, h=264, distance=3.0, gaborish=1, epf=2, kind="smooth", hdr="pq10000"),
    dict(w=300, h=520, distance=0.5, gaborish=1, epf=1, hdr="edges"),
    dict(w=333, h=277, distance=2.0, gaborish=1, epf=3, hdr=5),
])
def test_frames_stage_by_stage(cfg, refmod):
    """Every stage prefix, hot path only, same coefficients: the reference's own
    DecodeGroupForRoundtrip + stages vs the C restatement. rcp_mode 1 (host rcpss, what the
    reference's AVX2 path executes on this machine) must be bit-exact; rcp_mode 0 (exact
    reciprocal = what the CUDA path computes) within 2e-5 absolute.  `hdr`: jxl_workload.header_params
    written into the opened frame (Frame.set_params); there the 2e-5 bound is checked on the XYB taps
    only: the 12-bit reciprocal's error reaches linear light through 3 g^2 times the opsin matrix, which
    these headers (brighter matrices, intensity target 80) raise several-fold."""
    from oracle import cpu
    cfg = dict(cfg)
    kind = cfg.pop("kind", "photo")
    hdr = cfg.pop("hdr", None)
    img = wl.synth_image(cfg["w"], cfg["h"], 77, kind)
    data = refmod.encode_rgb8(img, cfg["distance"], 7, cfg["gaborish"], cfg["epf"], 2)
    fr = refmod.Frame(data, 2)
    if hdr is not None:
        set_header(refmod, fr, hdr)
    d = fr.dump()
    desc = cpu.desc_from_dump(d, out_format=abi.OUT_PLANAR_F32)
    frame_mask = (1 if d.info.gab else 0) | (2 if d.info.epf_iters >= 3 else 0) | \
        (4 if d.info.epf_iters >= 1 else 0) | (8 if d.info.epf_iters >= 2 else 0)
    masks = [0, 16, frame_mask, frame_mask | 16]
    if d.info.epf_iters > 0:
        masks += [1, 1 | 4, 2 | 4 | 8]
    for mask in sorted(set(masks)):
        want, _ = fr.render(mask)
        desc.stage_mask = abi.STAGE_EXPLICIT | mask
        got1 = cpu.render_frame(desc, d.coeffs, rcp_mode=1)
        assert np.array_equal(got1, want), (mask, float(np.abs(got1 - want).max()))
        if hdr is None or not mask & 16:
            got0 = cpu.render_frame(desc, d.coeffs, rcp_mode=0)
            assert np.abs(got0 - want).max() <= 2e-5, mask
    if hdr is not None:      # (the public decoder reads the header from the bitstream)
        fr.close()
        return
    # and the full public-API decode of the default-flag build (compiler-made FMAs differ)
    refmod.use_variant("default")
    full = refmod.decode_linear_f32(data, 1)
    refmod.use_variant("strict")
    desc.stage_mask = 0
    desc.out_format = abi.OUT_RGB_F32
    got = cpu.render_frame(desc, d.coeffs, rcp_mode=0)
    assert np.abs(got - full).max() <= 5e-5
    fr.close()


def test_hot_path_render_equals_public_decode(refmod):
    """The transform-only CPU baseline (ref_frame_render) is the same computation the public
    decoder does after entropy decoding: identical pixels."""
    refmod.use_variant("default")
    try:
        img = wl.synth_image(520, 300, 5)
        data = refmod.encode_rgb8(img, 1.0, 7, -1, -1, 2)
        full = refmod.decode_linear_f32(data, 2)
        fr = refmod.Frame(data, 2)
        planar, secs = fr.render(-1, reps=2)
        assert np.array_equal(planar.transpose(1, 2, 0), full)
        assert len(secs) == 2 and all(s > 0 for s in secs)
        fr.close()
    finally:
        refmod.use_variant("strict")


@pytest.mark.parametrize("fmt,srgb,hdr", [
    *[pytest.param(f, s, None, id=f"{f}-{s}") for f, s in [
        (abi.OUT_RGB_F32, True), (abi.OUT_RGB_U8, True), (abi.OUT_RGBA_U8, True), (abi.OUT_RGB_U16, True),
        (abi.OUT_RGB_F16, True), (abi.OUT_RGB_U8, False), (abi.OUT_RGB_F16, False)]],
    # non-default headers written into the reference's frame state (Frame.set_params)
    (abi.OUT_RGB_U8, True, "pq10000"), (abi.OUT_RGBA_U8, True, "dim80"), (abi.OUT_RGB_U16, True, "edges"),
    (abi.OUT_RGB_F16, False, "dim80"), (abi.OUT_RGB_F32, True, 11)])
def test_output_stages_bit_exact(fmt, srgb, hdr, refmod):
    """FromLinearStage<OpRgb> + WriteToOutputStage (dithered u8, RGBA, u16, binary16, f32) of the strict
    reference build vs the restatement, whole frame, host-rcpss mode: identical bytes."""
    from oracle import cpu
    img = wl.synth_image(333, 277, 5)
    data = refmod.encode_rgb8(img, 1.0, 7, -1, 2, 2)
    fr = refmod.Frame(data, 2)
    if hdr is not None:
        set_header(refmod, fr, hdr)
    d = fr.dump()
    want, _ = fr.render_out(-33 if srgb else -1, fmt)
    desc = cpu.desc_from_dump(d, out_format=fmt, stage_mask=abi.STAGE_SRGB if srgb else 0)
    got = cpu.render_frame(desc, d.coeffs, rcp_mode=1)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(got.view(np.uint16) if got.dtype == np.float16 else got,
                          want.view(np.uint16) if want.dtype == np.float16 else want)
    fr.close()


@pytest.mark.parametrize("xs,ys", [(256, 256), (960, 540), (37, 21)])
def test_dc_stage_bit_exact(xs, ys, refmod):
    """DequantDC + AdaptiveDCSmoothing of the reference (both builds) vs the restatement."""
    from oracle import cpu
    q = support.dc_stage_input(xs, ys)
    for variant in ("strict", "default"):
        refmod.use_variant(variant)
        try:
            for mul in (1.0, 0.5):
                assert np.array_equal(refmod.dequant_dc(q, support.DC_FACTORS, mul, support.DC_CFL),
                                      cpu.dequant_dc(q, support.DC_FACTORS, mul, support.DC_CFL))
            dc = cpu.dequant_dc(q, support.DC_FACTORS, 1.0, support.DC_CFL)
            assert np.array_equal(refmod.adaptive_dc_smoothing(dc, support.DC_FACTORS, 3),
                                  cpu.adaptive_dc_smoothing(dc, support.DC_FACTORS))
        finally:
            refmod.use_variant("strict")


@pytest.mark.parametrize("fmt,dtype,ch", [(abi.OUT_RGB_U8, np.uint8, 3), (abi.OUT_RGBA_U8, np.uint8, 4),
                                          (abi.OUT_RGB_U16, np.uint16, 3), (abi.OUT_RGB_F16, np.float16, 3),
                                          (abi.OUT_RGB_F32, np.float32, 3)])
def test_full_chain_equals_default_public_decode(fmt, dtype, ch, refmod):
    """The path with JXLGPU_STAGE_SRGB and a packed output format is, byte for byte, what the reference's
    PUBLIC decoder delivers by default for an sRGB image (what `djxl in.jxl out.png` writes): public API
    == hot path + FromLinear + WriteToOutput (reference stages) == the restatement (strict build)."""
    from oracle import cpu
    img = wl.synth_image(333, 277, 5)
    data = refmod.encode_rgb8(img, 1.0, 7, -1, -1, 2)
    public = refmod.decode_native(data, (277, 333, ch), dtype, 2)
    fr = refmod.Frame(data, 2)
    d = fr.dump()
    hot, _ = fr.render_out(-33, fmt)
    fr.close()
    desc = cpu.desc_from_dump(d, out_format=fmt, stage_mask=abi.STAGE_SRGB)
    restated = cpu.render_frame(desc, d.coeffs, rcp_mode=1)

    def bits(a):
        return a.view(np.uint16) if a.dtype == np.float16 else a
    assert np.array_equal(bits(public), bits(hot))
    assert np.array_equal(bits(public), bits(restated))
    # and it is a decode of the image that went in (8-bit sRGB in, d1.0): mean abs error < 2 %
    scale = {np.uint8: 255.0, np.uint16: 65535.0}.get(dtype, 1.0)
    assert np.abs(public[..., :3].astype(np.float64) / scale - img / 255.0).mean() < 0.02


@pytest.mark.parametrize("distance", [1.0, 8.0])
def test_group_major_ac_image_is_a_drop_in(distance, refmod):
    """integration/pinned_ac_image.h (the storage class a libjxl host installs for a GPU frame) driven by
    the UNMODIFIED reference decoder through libjxl's abstract ACImage interface: same coefficients,
    same pixels, and the allocation is the [group][channel][65536] layout the C ABI takes as is."""
    img = wl.synth_image(600, 300, 21)
    data = refmod.encode_rgb8(img, distance, 7, -1, -1, 2)
    a = refmod.Frame(data, 2)
    b = refmod.Frame(data, 2, storage=1)
    da, db = a.dump(), b.dump()
    assert da.coeffs.dtype == db.coeffs.dtype and np.array_equal(da.coeffs, db.coeffs)
    assert np.array_equal(da.decoded, db.decoded)
    raw = b.raw_group_major_coeffs()
    assert raw.shape == (da.info.num_groups, 3, 65536)
    assert np.array_equal(raw.transpose(1, 0, 2), da.coeffs)
    assert np.count_nonzero(raw) > 0
    a.close()
    b.close()


@pytest.mark.parametrize("cfg", [dict(w=517, h=331, distance=1.0, gaborish=1, epf=3), dict(w=300, h=520, distance=0.5, gaborish=0, epf=0),
                                 dict(w=517, h=331, distance=1.0, gaborish=1, epf=3, hdr="dim80"),
                                 dict(w=300, h=520, distance=0.5, gaborish=1, epf=2, hdr="edges")])
def test_gpu_frame_binding_from_decoder_state(cfg, refmod):
    """integration/gpu_frame_binding.h -- the C++ a libjxl maintainer adds to fill jxlgpu_frame from
    PassesDecoderState -- applied to the unmodified reference's live decoder state: every scalar equals
    the description the tests build by hand, and the oracle rendered straight from the bound struct
    (zero-copy pointers + strides into libjxl's images) gives the reference's pixels.  With `hdr` the frame
    state carries a non-default header whose per-channel values all differ: every header field of the bound
    struct equals the value written, which pins the binding's field mapping."""
    import ctypes as C
    from oracle import cpu
    img = wl.synth_image(cfg["w"], cfg["h"], 31)
    data = refmod.encode_rgb8(img, cfg["distance"], 7, cfg["gaborish"], cfg["epf"], 2)
    fr = refmod.Frame(data, 2)
    hdr = wl.header_params(cfg["hdr"]) if "hdr" in cfg else None
    if hdr is not None:
        set_header(refmod, fr, cfg["hdr"])
    d = fr.dump()
    bound = fr.bind_gpu_frame(abi.OUT_RGB_F32, 0)
    if hdr is not None:
        for name in wl.HEADER_FIELDS:
            got = np.float32(list(getattr(bound, name)) if hasattr(getattr(bound, name), "__len__") else getattr(bound, name))
            assert np.array_equal(got, np.float32(hdr[name])), name
    by_hand = cpu.desc_from_dump(d).to_struct()
    pointer_fields = {"ac_strategy", "raw_quant", "epf_sharpness", "ytox_map", "ytob_map", "dc", "dequant_table",
                      "quant_dc", "dc_group_mul"}
    stride_fields = {"ac_strategy_stride", "raw_quant_stride", "epf_sharpness_stride", "cmap_stride", "dc_stride"}
    for name, _ in abi.JxlGpuFrame._fields_:
        if name in pointer_fields or name in stride_fields:
            continue
        a, b = getattr(bound, name), getattr(by_hand, name)
        if hasattr(a, "__len__"):
            assert list(a) == list(b), name
        else:
            assert a == b, name
    assert bound.raw_quant_stride >= bound.xsize_blocks and bound.dc_stride >= bound.xsize_blocks
    # render with the oracle straight from the bound struct
    co = np.ascontiguousarray(d.coeffs)
    ptrs = (C.c_void_p * 3)(*[co.ctypes.data + c * co[0].nbytes for c in range(3)])
    out = np.zeros((d.info.ysize, d.info.xsize, 3), np.float32)
    assert cpu.lib().jxo_render_frame(C.byref(bound), ptrs, 1, out.ctypes.data) == 0
    want, _ = fr.render(-1)
    assert np.array_equal(out, want.transpose(1, 2, 0))
    fr.close()


@pytest.mark.parametrize("rs,w,h", [(2, 600, 300), (4, 1100, 210), (8, 2100, 160)])
def test_upsampling_stage_bit_exact(rs, w, h, refmod):
    """SURVEY.md §8f rank 4, UpsamplingStage (stage_upsampling.cc:51-271): frames encoded with resampling 2/4/8.
    The restatement (jxo_upsample_plane, after the filters and before XYB like PreparePipeline orders them) is
    bit-exact against the reference's own stage, and the reference's hot path + stage equals its public decode."""
    from oracle import cpu
    img = wl.synth_image(w, h, seed=rs)
    data = refmod.encode_rgb8(img, 1.0, 7, -1, -1, 4, resampling=rs)
    fr = refmod.Frame(data, 2)
    i = fr.info
    assert i.upsampling == rs and (i.xsize_upsampled, i.ysize_upsampled) == (w, h)
    d = fr.dump()
    desc = cpu.desc_from_dump(d)
    assert desc.upsampling == rs and desc.out_xsize == w and desc.out_ysize == h
    desc.out_format = abi.OUT_PLANAR_F32
    chain = (1 if i.gab else 0) | (2 if i.epf_iters >= 3 else 0) | (4 if i.epf_iters >= 1 else 0) | (8 if i.epf_iters >= 2 else 0)
    want, _ = fr.render(chain | refmod.STAGE_XYB | refmod.STAGE_UPSAMPLING)
    assert want.shape == (3, h, w)
    got = cpu.render_frame(desc, d.coeffs, rcp_mode=1)
    assert np.array_equal(got, want)
    desc.stage_mask = abi.STAGE_EXPLICIT | chain          # the upsampled XYB planes themselves
    want_xyb, _ = fr.render(chain | refmod.STAGE_UPSAMPLING)
    assert np.array_equal(cpu.render_frame(desc, d.coeffs, rcp_mode=1), want_xyb)
    fr.close()
    full = refmod.decode_linear_f32(data, 2)              # the decoder's real pipeline
    assert np.array_equal(np.moveaxis(want, 0, 2), full)


@pytest.mark.parametrize("rs,w,h,iso,hdr", [
    *[pytest.param(*c, None, id="-".join(map(str, c))) for c in [(1, 600, 300, 3200), (2, 600, 299, 6400), (1, 523, 260, 1600)]],
    (1, 600, 300, 3200, "pq10000"), (2, 600, 299, 6400, "edges"), (1, 523, 260, 1600, "dim80")])
def test_noise_stages_bit_exact(rs, w, h, iso, hdr, refmod):
    """SURVEY.md §8f rank 4, noise: frames the reference encoder made with photon noise (frame flag kNoise).
    Random3Planes (dec_noise.cc:45-152) + ConvolveNoiseStage + AddNoiseStage (stage_noise.cc) restated in
    oracle/jxl_oracle.c: bit-exact against the reference's own stages, alone and behind the upsampling, and the
    reference's hot path + stages equals its public decode.  `hdr`: a non-default header (CfL base correlations
    included, which AddNoise reads) written into the reference's frame state."""
    from oracle import cpu
    img = wl.synth_image(w, h, seed=rs + iso)
    data = refmod.encode_rgb8(img, 1.0, 7, -1, -1, 4, resampling=rs | ((iso // 100) << 16))
    fr = refmod.Frame(data, 2)
    if hdr is not None:
        set_header(refmod, fr, hdr)
        assert fr.info.cfl_base_x != 0 and fr.info.cfl_base_b not in (0.0, 1.0)
    i = fr.info
    assert i.noise == 1 and max(i.noise_lut) > 1e-3 and i.upsampling == rs
    d = fr.dump()
    desc = cpu.desc_from_dump(d)
    assert desc.noise == 1 and (desc.visible_frame_index, desc.nonvisible_frame_index) == (1, 0)
    desc.out_format = abi.OUT_PLANAR_F32
    chain = (1 if i.gab else 0) | (2 if i.epf_iters >= 3 else 0) | (4 if i.epf_iters >= 1 else 0) | (8 if i.epf_iters >= 2 else 0)
    want, _ = fr.render(chain | refmod.STAGE_XYB | refmod.STAGE_UPSAMPLING | refmod.STAGE_NOISE)
    assert np.array_equal(cpu.render_frame(desc, d.coeffs, rcp_mode=1), want)
    without, _ = fr.render(chain | refmod.STAGE_XYB | refmod.STAGE_UPSAMPLING)
    assert not np.array_equal(without, want)
    fr.close()
    if hdr is None:      # (the public decoder reads the header from the bitstream)
        assert np.array_equal(np.moveaxis(want, 0, 2), refmod.decode_linear_f32(data, 2))


def need_ups_noise_setters(refmod):
    """Frame.set_upsampling_weights / set_noise_lut; a harness prebuilt without them is a skip only where the
    reference sources are not there to rebuild it."""
    import os
    if not refmod.can_set_ups_noise():
        if os.path.isdir(os.environ.get("JXL_REFERENCE_ROOT", "/root/reference")):
            pytest.fail("oracle/_ref predates ref_frame_set_upsampling_weights / ref_frame_set_noise_lut although the "
                        "reference is present: run `python oracle/build_ref.py`")
        pytest.skip("oracle/_ref was built from a harness without ref_frame_set_upsampling_weights")


@pytest.mark.parametrize("rs,w,h,noise,hdr", [(2, 601, 299, False, None), (4, 1101, 517, False, None),
                                              (8, 2101, 167, False, None), (4, 1101, 517, True, None),
                                              (8, 2101, 167, True, None), (8, 2101, 167, True, "edges")])
def test_custom_weights_and_noise_lut_bit_exact(rs, w, h, noise, hdr, refmod):
    """Random F16 upsampling weights (negative ones, no two entries of the triangular layout related:
    support.custom_upsampling_weights) read into the reference's CustomTransformData through its Bundle reader, and
    the wide non-monotone LUT (support.NOISE_LUT_WIDE, up to 1023/1024) through its DecodeNoise.  Output sizes are
    multiples of neither N nor 16 nor 256, so noise tiles and the upsampler's mirror are ragged.  The oracle is
    bit-exact against the reference's own stages, with and without the colour stage; the weights really are the
    custom ones (the render differs from the default weights')."""
    import dataclasses
    from oracle import cpu
    need_ups_noise_setters(refmod)
    img = wl.synth_image(w, h, seed=rs + 7)
    data = refmod.encode_rgb8(img, 1.0, 7, -1, -1, 4, resampling=rs | ((6400 // 100) << 16 if noise else 0))
    fr = refmod.Frame(data, 2)
    if hdr is not None:
        set_header(refmod, fr, hdr)
    wts = support.custom_upsampling_weights(rs, seed=rs + (1 if noise else 0))
    fr.set_upsampling_weights(rs, wts)
    if noise:
        fr.set_noise_lut(support.NOISE_LUT_WIDE)
    i = fr.info
    assert i.upsampling == rs and (i.xsize_upsampled, i.ysize_upsampled) == (w, h) and i.noise == int(noise)
    assert np.array_equal(np.float32(list(i.upsampling_weights)[:support.UPS_WEIGHT_COUNT[rs]]), wts)
    if noise:
        assert np.array_equal(np.float32(list(i.noise_lut)), np.float32(support.NOISE_LUT_WIDE))
    d = fr.dump()
    desc = cpu.desc_from_dump(d)
    desc.out_format = abi.OUT_PLANAR_F32
    chain = (1 if i.gab else 0) | (2 if i.epf_iters >= 3 else 0) | (4 if i.epf_iters >= 1 else 0) | (8 if i.epf_iters >= 2 else 0)
    stages = refmod.STAGE_UPSAMPLING | (refmod.STAGE_NOISE if noise else 0)
    want, _ = fr.render(chain | refmod.STAGE_XYB | stages)
    assert want.shape == (3, h, w)
    got = cpu.render_frame(desc, d.coeffs, rcp_mode=1)
    assert np.array_equal(got, want)
    desc.stage_mask = abi.STAGE_EXPLICIT | chain          # the upsampled (noisy) XYB planes themselves
    want_xyb, _ = fr.render(chain | stages)
    assert np.array_equal(cpu.render_frame(desc, d.coeffs, rcp_mode=1), want_xyb)
    ups_xyb, _ = fr.render(chain | refmod.STAGE_UPSAMPLING)
    fr.close()
    default = dataclasses.replace(desc, upsampling_weights=support.default_upsampling_weights(rs), noise=0)
    assert not np.array_equal(cpu.render_frame(default, d.coeffs, rcp_mode=1), ups_xyb)
    if noise:   # what AddNoise sees: content of an 8-bit sRGB image keeps Y +- X below 7/3, short of saturation
        X, Y = ups_xyb[0].astype(np.float64), ups_xyb[1].astype(np.float64)
        seg = np.concatenate([support.lut_segments((Y - X) * 0.5).ravel(), support.lut_segments((Y + X) * 0.5).ravel()])
        counts = np.bincount(seg + 1, minlength=9)
        print(f"{rs}x {w}x{h}: AddNoise inputs per LUT branch (negative, segments 0..6, saturated): {counts.tolist()}")
        assert (counts[1:4] >= 100).all(), counts


def make_jpeg(w, h, quality, seed=5):
    """A baseline 4:4:4 JPEG of the seeded test image (Pillow)."""
    import io
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(wl.synth_image(w, h, seed)).save(b, format="JPEG", quality=quality, subsampling=0)
    return b.getvalue()


@pytest.mark.parametrize("w,h,q", [(600, 300, 90), (517, 331, 75)])
def test_jpeg_origin_ycbcr_frames(w, h, q, refmod):
    """SURVEY.md §8f rank 4, YCbCr: a 4:4:4 JPEG recompressed by the reference encoder (JxlEncoderAddJPEGFrame) is a
    VarDCT frame with the YCbCr colour transform.  Dequantisation + IDCT are the XYB path's; the colour stage is
    kYCbCrStage (stage_ycbcr.cc:33-71).  Restatement bit-exact against the reference's stages, and its 8-bit output
    identical to the reference's PUBLIC decoder (no transfer function follows: the image is not XYB-encoded)."""
    pytest.importorskip("PIL")
    from oracle import cpu
    data = refmod.encode_jpeg(make_jpeg(w, h, q), 4)
    fr = refmod.Frame(data, 2)
    i = fr.info
    assert i.ycbcr == 1 and i.gab == 0 and i.epf_iters == 0
    d = fr.dump()
    desc = cpu.desc_from_dump(d)
    assert desc.color_transform == 1
    desc.out_format = abi.OUT_PLANAR_F32
    want, _ = fr.render(refmod.STAGE_XYB)          # bit 16 = the frame's colour transform
    fr.close()
    assert np.array_equal(cpu.render_frame(desc, d.coeffs, rcp_mode=1), want)
    desc.out_format = abi.OUT_RGB_U8
    assert np.array_equal(cpu.render_frame(desc, d.coeffs, rcp_mode=1), refmod.decode_native(data, (h, w, 3), np.uint8, 2))
