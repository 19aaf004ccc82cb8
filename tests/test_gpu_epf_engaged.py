"""-m gpu: the edge-preserving filter where it engages, at the sizes where its scheduling and tiling run.

synthetic_frame draws quantisers 1..256, so the EPF changes about 0.1 % of its pixels and almost none next to a
group-row boundary: band halos, the streaming scheduler's neighbour rule, the strip kernel's block permutation over
long segments and the fused kernel's persistent units would all pass with the EPF switched off.  Every frame here is
support.epf_frame, whose oracle EPF coverage (pixels the chain's EPF passes change) is asserted and printed: a few
hundred changed pixels around every group-row boundary, something in every 64-row and every 240-column window.

Device buffers only grow and are never cleared, so a kernel that reads a row before it is written would read that
frame's correct values from the last render of the same frame.  Every checked render here therefore follows a decoy
frame on the same context (support.decoy_frame: same geometry, other content, EPF engaged on every block).

Bar: bit-exact against oracle/jxl_oracle.c in exact-reciprocal mode; the float64 model of EPF passes 0 / 1 / 2 at
the end checks the GPU's tile-kernel taps within a bound counted from float32 operations."""
import dataclasses

import numpy as np
import pytest

from libjxl_b200 import abi, pipeline, sharding
from tests import support

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("built")]

CHAINS = {20: (0, 1), 21: (1, 1), 28: (0, 2), 29: (1, 2), 30: (0, 3), 31: (1, 3)}   # stage mask: (gab, epf_iters)
FUSED = (20, 21, 28, 29, 30)
F32 = (abi.OUT_RGB_F32, 0)
SRGB8 = (abi.OUT_RGB_U8, abi.STAGE_SRGB)
FRAMES = {"4k": (3840, 2160, abi.AC_INT16), "8k": (7680, 4320, abi.AC_INT32), "bands": (1500, 2300, abi.AC_INT16),
          "ragged": (1231, 1021, abi.AC_INT16)}


@pytest.fixture(scope="module")
def cache():
    store = {}
    yield store
    store.clear()


def frame(cache, name, chain, fmt=F32):
    """(desc, coeffs, oracle image) of FRAMES[name] under stage chain `chain` and output `fmt`; the EPF coverage of
    the chain is asserted the first time the frame is asked for in f32."""
    if ("base", name) not in cache:
        w, h, ac = FRAMES[name]
        cache[("base", name)] = support.epf_frame(w, h, seed=w + h, ac_type=ac)
    key = (name, chain, fmt)
    if key not in cache:
        from oracle import cpu
        desc, coeffs = cache[("base", name)]
        gab, iters = CHAINS[chain]
        desc = dataclasses.replace(desc, gab=gab, epf_iters=iters, out_format=fmt[0], stage_mask=fmt[1])
        want = cpu.render_frame(desc, coeffs, rcp_mode=0)
        if fmt == F32:
            nogab = ("noepf", name, gab)
            if nogab not in cache:
                cache[nogab] = cpu.render_frame(support.without_epf(desc), coeffs, rcp_mode=0)
            mask = support.changed_pixels(want, cache[nogab], False)
            bands = {y for world in (2, 3, 4, 8) for y0, _ in sharding.band_partition(desc.ysize_groups, world)
                     for y in [y0 * abi.GROUP_DIM] if 0 < y < desc.ysize}
            support.assert_epf_coverage(mask, f"{name} chain {chain}", band_rows=bands)
        cache[key] = desc, coeffs, want
    return cache[key]


def context(monkeypatch, fused=False, launch_mb=None, generic=False):
    """A new context: JXLGPU_FUSED / JXLGPU_LAUNCH_MB / JXLGPU_FORCE_GENERIC_FILTER are read when it is created."""
    monkeypatch.setenv("JXLGPU_FUSED", "1" if fused else "0")
    monkeypatch.setenv("JXLGPU_FORCE_GENERIC_FILTER", "1" if generic else "0")
    if launch_mb is None:
        monkeypatch.delenv("JXLGPU_LAUNCH_MB", raising=False)
    else:
        monkeypatch.setenv("JXLGPU_LAUNCH_MB", str(launch_mb))
    return pipeline.TransformPipeline(device=0, num_host_threads=2)


def assert_same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, what
    if not np.array_equal(got, want):
        d = got.astype(np.float64) != want.astype(np.float64)
        rows = np.nonzero(d.reshape(d.shape[0], -1).any(1))[0]
        raise AssertionError(f"{what}: {int(d.sum())} of {d.size} samples differ, in rows {rows.min()}..{rows.max()}")


def render_resident(p, desc, coeffs):
    """set_device_coefficients + frame_begin + render_device into a device buffer.  Returns (pixels, launches)."""
    import torch
    dev = torch.from_numpy(np.ascontiguousarray(coeffs)).cuda()
    rows = sharding.band_pixel_rows(desc, desc.band_y0_groups, desc.band_ny_groups)[1] if desc.band_ny_groups \
        else desc.ysize
    tdt = {np.dtype(np.float32): torch.float32, np.dtype(np.uint8): torch.uint8}[np.dtype(desc.out_dtype)]
    out = torch.zeros(desc.out_shape(rows), dtype=tdt, device="cuda")
    p.set_device_coefficients([dev[c].data_ptr() for c in range(3)])
    try:
        p.frame_begin(desc)
        before = p.launch_count()
        p.render_device(out.data_ptr(), desc.out_row_bytes, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        launches = p.launch_count() - before
    finally:
        p.set_device_coefficients(None)
    got = out.cpu().numpy()
    del out, dev
    return got, launches


def decoy(cache, p, desc, want, resident, k=0):
    """Render the decoy of `desc` (whole frame) on `p` and check it differs from the target almost everywhere."""
    key = ("decoy", desc.xsize, desc.ysize, desc.ac_type, desc.gab, desc.epf_iters, desc.out_format, desc.stage_mask, k)
    if key not in cache:
        cache[key] = support.decoy_frame(dataclasses.replace(desc, band_y0_groups=0, band_ny_groups=0),
                                         seed=desc.xsize + 17 * k + 1)
    d, c = cache[key]
    px = render_resident(p, d, c)[0] if resident else p.decode_frame(d, c)
    support.assert_decoy_differs(px, want, False)


# ---- production chains at 4K, device-resident ----
CASES_4K = [(m, False, F32) for m in CHAINS] + [(m, True, F32) for m in FUSED] + \
           [(21, False, SRGB8), (31, False, SRGB8), (21, True, SRGB8)]


@pytest.mark.parametrize("chain,fused,fmt", CASES_4K,
                         ids=[f"{m}-{'fused' if f else 'two-kernel'}-{'srgb8' if o == SRGB8 else 'f32'}" for m, f, o in CASES_4K])
def test_4k_production_chains(cache, monkeypatch, chain, fused, fmt):
    """3840x2160, EPF engaged on about half the blocks: strip kernel segments far beyond 64 rows (the permutation
    ring of EPF block rows turns over many times) and the fused kernel's persistent CTAs."""
    desc, coeffs, want = frame(cache, "4k", chain, fmt)
    if fmt != F32:
        frame(cache, "4k", chain)                 # (coverage of the chain)
    p = context(monkeypatch, fused=fused)
    try:
        decoy(cache, p, desc, want, resident=True)
        got, launches = render_resident(p, desc, coeffs)
    finally:
        p.close()
    assert launches == (5 if fused else 6)
    assert_same(got, want, f"chain {chain}")


def fused_units(desc, num_sms, forced_segs=None):
    """Work units of one launch of the fused kernel over the whole frame.  Mirrors launch_fused_mask in
    libjxl_b200/csrc/jxl_fused_inst.cu: strips of 240 columns times the row-segment count that maximises the
    efficiency estimate (segments of at least 96 rows, rounded up to whole blocks)."""
    mask = 16 | (abi.STAGE_GAB if desc.gab else 0) | (abi.STAGE_EPF0 if desc.epf_iters >= 3 else 0) | \
        (abi.STAGE_EPF1 if desc.epf_iters >= 1 else 0) | (abi.STAGE_EPF2 if desc.epf_iters >= 2 else 0)
    nst = max(1, bin(mask & 15).count("1"))
    band_h, strips = desc.ysize, (desc.xsize + 239) // 240
    best, best_segs = -1.0, 1
    for segs in range(1, 65):
        seg_rows = ((band_h + segs - 1) // segs + 7) & ~7
        if segs > 1 and seg_rows < 96:
            break
        real = (band_h + seg_rows - 1) // seg_rows
        units = strips * real
        rounds = (units + num_sms - 1) // num_sms
        eff = units / (rounds * num_sms) * seg_rows / (seg_rows + 8.0 * (nst + 2))
        if eff > best:
            best, best_segs = eff, real
    if forced_segs is not None:                  # JXLGPU_FUSED_SEGS
        best_segs = max(1, forced_segs)
    seg_rows = ((band_h + best_segs - 1) // best_segs + 7) & ~7
    return strips * ((band_h + seg_rows - 1) // seg_rows)


@pytest.mark.parametrize("chain,fused", [(21, False), (21, True), (31, False)],
                         ids=["21-two-kernel", "21-fused", "31-two-kernel"])
def test_8k_int32(cache, monkeypatch, chain, fused):
    """7680x4320 int32 (chain 21 is the benchmark's).  The fused launch sizes its row segments to fill one round of
    the grid (128 units on 132 SMs here), so the fused case asks for 8 segments: every CTA then runs several units,
    carrying its rings and sigma rows from one unit to the next."""
    import torch
    desc, coeffs, want = frame(cache, "8k", chain)
    if fused:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        monkeypatch.setenv("JXLGPU_FUSED_SEGS", "8")
        units = fused_units(desc, sms, forced_segs=8)
        print(f"8k chain {chain}: {fused_units(desc, sms)} fused units by default, {units} with 8 segments, {sms} SMs")
        assert units > sms, (units, sms)
    p = context(monkeypatch, fused=fused)
    try:
        decoy(cache, p, desc, want, resident=True)
        got, launches = render_resident(p, desc, coeffs)
    finally:
        p.close()
    assert launches == (5 if fused else 6)
    assert_same(got, want, f"8k chain {chain}")


# ---- bands ----
@pytest.mark.parametrize("fused", [False, True], ids=["two-kernel", "fused"])
@pytest.mark.parametrize("chain,fmt", [(31, F32), (31, SRGB8), (21, F32), (21, SRGB8)],
                         ids=["31-f32", "31-srgb8", "21-f32", "21-srgb8"])
def test_bands_after_decoys(cache, monkeypatch, chain, fmt, fused):
    """1500x2300 (9 group rows) in bands of world 2, 3, 4 and 8 ranks (8: one-row bands, the halo reaches into both
    neighbours), host-fed with only sharding.groups_needed and device-resident, each band after a decoy.  The
    concatenated bands are the oracle's frame (8-bit: the dither row depends on the band offset)."""
    if fused and chain == 31:
        pytest.skip("chain 31 has no fused kernel")
    desc, coeffs, want = frame(cache, "bands", chain, fmt)
    frame(cache, "bands", chain)
    p = context(monkeypatch, fused=fused)
    try:
        for world in (2, 3, 4, 8):
            for resident in (False, True):
                rows = []
                for i, (y0, ny) in enumerate(sharding.band_partition(desc.ysize_groups, world)):
                    decoy(cache, p, desc, want, resident, k=i % 2)
                    d = dataclasses.replace(desc, band_y0_groups=y0, band_ny_groups=ny)
                    if resident:
                        rows.append(render_resident(p, d, coeffs)[0])
                        continue
                    p.set_device_coefficients(None)
                    p.frame_begin(d)
                    for g in sharding.groups_needed(d, y0, ny):
                        p.submit_group(g, [coeffs[c, g] for c in range(3)])
                    rows.append(p.frame_finish())
                assert_same(np.concatenate(rows, axis=0), want,
                            f"world {world}, {'device-resident' if resident else 'host-fed'}")
    finally:
        p.close()


# ---- streaming ----
@pytest.mark.parametrize("launch_mb", [None, 0], ids=["default", "launch-mb-0"])
@pytest.mark.parametrize("chain,fused", [(31, False), (21, True)], ids=["31-two-kernel", "21-fused"])
def test_streaming_after_decoys(cache, monkeypatch, chain, fused, launch_mb):
    """Three shuffled submission orders with rows streamed back on and off, dense and sparse, on a context with the
    default launch size and one that launches every group row as soon as it is complete: a group row may be filtered
    only once its neighbours are transformed.  Each render follows a decoy."""
    desc, coeffs, want = frame(cache, "bands", chain)
    rng = np.random.default_rng(chain)
    p = context(monkeypatch, fused=fused, launch_mb=launch_mb)
    try:
        for sparse in (False, True):
            for trial in range(3):
                order = rng.permutation(desc.num_groups).tolist()
                decoy(cache, p, desc, want, resident=False, k=trial % 2)
                got = p.decode_frame(desc, coeffs, order=order, stream_output=trial % 2 == 0, sparse=sparse)
                assert_same(got, want, f"sparse={sparse} stream={trial % 2 == 0} order {order}")
    finally:
        p.close()


# ---- fused row segments, generic tile kernel ----
@pytest.mark.parametrize("segs", ["2", "5", None], ids=["segs2", "segs5", "default"])
def test_fused_row_segments(cache, monkeypatch, segs):
    """JXLGPU_FUSED_SEGS (read at every launch) cuts each strip into 2 or 5 row segments, or the launch picks its
    own: each segment re-transforms its halo block rows, and its boundaries must not show in the pixels."""
    if segs is None:
        monkeypatch.delenv("JXLGPU_FUSED_SEGS", raising=False)
    else:
        monkeypatch.setenv("JXLGPU_FUSED_SEGS", segs)
    p = context(monkeypatch, fused=True)
    try:
        for chain in FUSED:
            desc, coeffs, want = frame(cache, "ragged", chain)
            decoy(cache, p, desc, want, resident=True)
            got, launches = render_resident(p, desc, coeffs)
            assert launches == 5
            assert_same(got, want, f"chain {chain}, segments {segs}")
    finally:
        p.close()


@pytest.mark.parametrize("name", ["4k", "ragged"])
def test_generic_tile_kernel(cache, monkeypatch, name):
    """JXLGPU_FORCE_GENERIC_FILTER=1 sends the production chains to the generic tile kernel."""
    p = context(monkeypatch, generic=True)
    try:
        for chain in (21, 31):
            desc, coeffs, want = frame(cache, name, chain)
            decoy(cache, p, desc, want, resident=True)
            got, launches = render_resident(p, desc, coeffs)
            assert launches == 6
            assert_same(got, want, f"{name} chain {chain}, generic filter")
    finally:
        p.close()


# ---- a float64 model of EPF passes 0, 1 and 2 ----
U = 2.0 ** -24                       # float32 unit roundoff
SADS0 = [(-2, 0), (-1, -1), (-1, 0), (-1, 1), (0, -2), (0, -1), (0, 1), (0, 2), (1, -1), (1, 0), (1, 1), (2, 0)]
PLUS = [(0, 0), (-1, 0), (0, -1), (1, 0), (0, 1)]
CROSS = [(-1, 0), (0, -1), (0, 1), (1, 0)]


def inv_sigma64(desc):
    """Per pixel: float64 1/sigma (ComputeSigma) of the pixel's block, (H, W)."""
    q = support.block_quant(desc).astype(np.float64)
    lut = np.array(desc.epf_sharp_lut, np.float64)[desc.epf_sharpness]
    sq = desc.epf_quant_mul / (desc.quant_scale * q * -1.1715728752538099024)
    s = np.minimum(sq * lut, -1e-4)
    inv = np.repeat(np.repeat(1.0 / s, 8, 0), 8, 1)
    return inv[:desc.ysize, :desc.xsize]


def epf64(desc, x, which, variant=None):
    """EPF pass `which` on planes x (3, H, W) in float64, over mirror-padded shifted planes.  Returns (out, bound,
    engaged, excluded, weights strictly inside (0, 1) / weights): bound is the first-order error of the float32
    computation at every pixel; `variant` makes the model wrong on purpose."""
    _, h, w = x.shape
    P = np.pad(x, ((0, 0), (4, 4), (4, 4)), mode="symmetric")
    sh = lambda dy, dx: P[:, 4 + dy:4 + dy + h, 4 + dx:4 + dx + w]          # noqa: E731
    scale = np.array(desc.epf_channel_scale, np.float64)
    if variant == "permuted":
        scale = scale[[1, 2, 0]]
    sm = {0: desc.epf_pass0_sigma_scale * 1.65, 1: 1.65, 2: desc.epf_pass2_sigma_scale * 1.65}[which]
    if variant == "pass0-scale" and which == 1:
        sm = desc.epf_pass0_sigma_scale * 1.65
    yy, xx = np.mgrid[0:h, 0:w]
    row_border, col_border = (yy % 8 == 0) | (yy % 8 == 7), (xx % 8 == 0) | (xx % 8 == 7)
    border = col_border if variant == "columns-only" else row_border | col_border
    s = inv_sigma64(desc)
    inv = s * np.where(border, sm * desc.epf_border_sad_mul, sm)
    engaged = s >= float(support.K_MIN_SIGMA)
    excluded = np.abs(s / float(support.K_MIN_SIGMA) - 1.0) <= 1e-5
    if which in (0, 1):
        taps = SADS0 if which == 0 else CROSS
        sads = [sum(scale[c] * sum(np.abs(sh(oy, ox)[c] - sh(dy + oy, dx + ox)[c]) for oy, ox in PLUS)
                    for c in range(3)) for dy, dx in taps]
        nterm = 15
    else:
        taps = CROSS
        sads = [sum(scale[c] * np.abs(sh(dy, dx)[c] - x[c]) for c in range(3)) for dy, dx in taps]
        nterm = 3
    k_sad = 2 * nterm + 2            # each |a - b| and each sum / fma rounds once, relative to the (positive) total
    k_sig = 8                        # quant_mul / (scale * q * num), * lut, 1 / sigma, * sm (* border mul), sm itself
    num = x.copy()
    wsum = np.ones((h, w))
    e_w = []
    absnum = np.abs(x).copy()
    inside = total = 0
    for (dy, dx), sad in zip(taps, sads):
        wt = np.maximum(0.0, 1.0 + sad * inv)
        num = num + wt * sh(dy, dx)
        absnum = absnum + wt * np.abs(sh(dy, dx))
        wsum = wsum + wt
        e_w.append((k_sad + k_sig) * U * np.abs(sad * inv) + U)    # Lipschitz 1 through max(0, .)
        inside += int(((wt > 0) & (wt < 1) & engaged).sum())
        total += int(engaged.sum())
    n = len(taps)
    out = num / wsum
    e_num = n * U * absnum + sum(e * np.abs(sh(dy, dx)) for (dy, dx), e in zip(taps, e_w))
    e_wsum = n * U * wsum + sum(e_w)
    bound = 2.0 * ((e_num + np.abs(out) * e_wsum) / wsum + 2 * U * np.abs(out))
    out = np.where(engaged, out, x)
    bound = np.where(engaged, bound, 0.0)
    return out, bound, engaged, excluded, inside / max(total, 1)


TAP_PAIRS = [(1, 3, 0), (3, 7, 1), (7, 15, 2), (0, 2, 0), (0, 4, 1), (0, 8, 2)]   # (input tap, output tap, pass)


@pytest.mark.parametrize("hdr", [None, "dim80"], ids=["default-header", "dim80"])
def test_float64_model_of_epf(hdr, monkeypatch):
    """The tile kernel's own taps (STAGE_EXPLICIT masks: Gaborish, then EPF 0, 1, 2, and each EPF pass alone after
    the transforms) against a float64 model of the pass applied to the GPU's input tap, within a bound counted from
    the float32 operations.  Blocks whose float64 inverse sigma is within 1e-5 of kMinSigma are left out (the
    float32 decision may go either way); they must be rare.  Three wrong models must break the bound."""
    desc, coeffs = support.epf_frame(1031, 517, seed=1031, hdr=hdr)
    p = context(monkeypatch)
    taps = {}
    try:
        for m in sorted({a for a, _, _ in TAP_PAIRS} | {b for _, b, _ in TAP_PAIRS}):
            d = dataclasses.replace(desc, stage_mask=abi.STAGE_EXPLICIT | m, out_format=abi.OUT_PLANAR_F32)
            taps[m] = p.decode_frame(d, coeffs).astype(np.float64)
    finally:
        p.close()
    for a, b, which in TAP_PAIRS:
        out, bound, engaged, excluded, inside = epf64(desc, taps[a], which)
        keep = ~excluded
        err = np.abs(taps[b] - out)[:, keep]
        ratio = float((err / np.maximum(bound[:, keep], 1e-300)).max())
        changed = float((taps[b] != taps[a]).any(0).mean())
        print(f"EPF{which} tap {a} -> {b}: {engaged.mean():.1%} of pixels engaged, {changed:.1%} changed, "
              f"{inside:.1%} of engaged weights in (0, 1), {int(excluded.sum())} pixels excluded, "
              f"max err / bound {ratio:.3f}, max bound {bound.max():.2e}")
        assert excluded.mean() < 1e-3
        assert changed > 0.05 and inside > 0.08
        assert (err <= bound[:, keep]).all(), (a, b, ratio)
        assert np.array_equal(taps[b][:, ~engaged], taps[a][:, ~engaged])
    for variant, (a, b, which) in (("pass0-scale", TAP_PAIRS[1]), ("columns-only", TAP_PAIRS[0]),
                                   ("permuted", TAP_PAIRS[5])):
        out, bound, _, excluded, _ = epf64(desc, taps[a], which, variant)
        err = np.abs(taps[b] - out)[:, ~excluded]
        assert (err > bound[:, ~excluded]).any(), f"the bound does not see the wrong model {variant}"
