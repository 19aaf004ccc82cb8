"""The edge-preserving filter where it engages, under the SIMT emulation of tests/emu (no GPU): frames on which the
EPF changes pixels along every group-row boundary (support.epf_frame), rendered in bands, streamed in shuffled order,
one launch per group row and in fused-kernel row segments, each render right after a decoy frame on the same
context so that a kernel reading a row before it is written shows it in the pixels.  Bit-exact against the oracle.
The GPU counterpart at 4K / 8K is tests/test_gpu_epf_engaged.py."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from libjxl_b200 import abi, pipeline, sharding
from tests import support

W, H = 300, 800          # 2 x 4 AC groups: bands of one group row have a neighbour on both sides
SRGB8 = (abi.OUT_RGB_U8, abi.STAGE_SRGB)
F32 = (abi.OUT_RGB_F32, 0)


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu import build_emu
    so = build_emu.build()
    saved = pipeline._lib
    pipeline._lib = pipeline.bind(C.CDLL(str(so)))      # the emulated library instead of libjxl_b200.so
    yield
    pipeline._lib = saved


def context(monkeypatch, fused=False, launch_mb=None):
    """A new emulated context: JXLGPU_FUSED / JXLGPU_LAUNCH_MB are read when it is created."""
    monkeypatch.setenv("JXLGPU_FUSED", "1" if fused else "0")
    if launch_mb is None:
        monkeypatch.delenv("JXLGPU_LAUNCH_MB", raising=False)
    else:
        monkeypatch.setenv("JXLGPU_LAUNCH_MB", str(launch_mb))
    return pipeline.TransformPipeline(device=0, num_host_threads=2)


_cache = {}


def frame(mask, fmt=F32):
    """support.epf_frame at W x H with stage chain `mask` (gab = bit 0, epf_iters 3 / 1 for chains 31 / 21) and an
    output layout, its oracle image, and its EPF coverage checked once."""
    key = (mask, fmt)
    if key not in _cache:
        from oracle import cpu
        gab, iters = mask & 1, {31: 3, 30: 3, 29: 2, 28: 2, 21: 1, 20: 1}[mask]
        desc, coeffs = support.epf_frame(W, H, seed=mask, gab=gab, epf_iters=iters)
        desc.out_format, desc.stage_mask = fmt
        want = cpu.render_frame(desc, coeffs, rcp_mode=0)
        if fmt == F32:
            # (+-7 rows of a 300-pixel row are 4200 pixels: 150 changed ones there are as dense as a few hundred at 1500)
            support.assert_epf_coverage(support.epf_coverage(desc, coeffs, with_epf=want), f"{W}x{H} chain {mask}",
                                        boundary_min=150)
        _cache[key] = desc, coeffs, want
    return _cache[key]


def decoy(p, desc, seed, want):
    """Render a decoy frame on `p` (whole frame, host-fed) and check it really differs from the target."""
    d, c = support.decoy_frame(dataclasses.replace(desc, band_y0_groups=0, band_ny_groups=0), seed)
    support.assert_decoy_differs(p.decode_frame(d, c), want, desc.out_format == abi.OUT_PLANAR_F32)


def same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, what
    if not np.array_equal(got, want):
        d = got.astype(np.float64) != want.astype(np.float64)
        rows = np.nonzero(d.reshape(d.shape[0], -1).any(1))[0]
        raise AssertionError(f"{what}: {int(d.sum())} samples differ, rows {rows.min()}..{rows.max()}")


def render_bands(p, desc, coeffs, want, world, resident, seed):
    """Every band of a `world`-rank partition, each after a decoy: host-fed with only the groups
    sharding.groups_needed names, or from device-resident planes.  Returns the concatenated bands."""
    rows = []
    dev = np.ascontiguousarray(coeffs)                      # "device" memory is host memory here
    for i, (y0, ny) in enumerate(sharding.band_partition(desc.ysize_groups, world)):
        if ny == 0:
            continue
        decoy(p, desc, seed + i, want)
        d = dataclasses.replace(desc, band_y0_groups=y0, band_ny_groups=ny)
        if resident:
            y, n = sharding.band_pixel_rows(d, y0, ny)
            out = np.zeros(d.out_shape(n), d.out_dtype)
            p.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
            try:
                p.frame_begin(d)
                p.render_device(out.ctypes.data, d.out_row_bytes)
                p.synchronize()
            finally:
                p.set_device_coefficients(None)
        else:
            p.set_device_coefficients(None)
            p.frame_begin(d)
            for g in sharding.groups_needed(d, y0, ny):
                p.submit_group(g, [coeffs[c, g] for c in range(3)])
            out = p.frame_finish()
        rows.append(out)
    return np.concatenate(rows, axis=0)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fused", [False, True], ids=["two-kernel", "fused"])
@pytest.mark.parametrize("mask,fmt", [(31, F32), (21, SRGB8)], ids=["chain31-f32", "chain21-srgb8"])
def test_emulated_epf_bands_after_decoys(emu_lib, monkeypatch, mask, fmt, fused):
    """Bands of two group rows and of one (world 4: the 7-row halo reaches into both neighbours), host-fed and
    device-resident, each band after a decoy: the concatenated bands are the oracle's frame."""
    desc, coeffs, want = frame(mask, fmt)
    p = context(monkeypatch, fused=fused)
    try:
        for world, resident in ((2, False), (4, False), (4, True)):
            got = render_bands(p, desc, coeffs, want, world, resident, seed=100 * world)
            same(got, want, f"world {world}, {'device-resident' if resident else 'host-fed'}")
    finally:
        p.close()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fused", [False, True], ids=["two-kernel", "fused"])
def test_emulated_epf_shuffled_streaming_after_decoys(emu_lib, monkeypatch, fused):
    """Groups in three shuffled orders (rows streamed back on alternate orders), the sparse hand-off, and a context
    that launches every group row as soon as it is complete (JXLGPU_LAUNCH_MB=0): the scheduler may filter a group
    row only once the rows above and below it are transformed.  Each render follows a decoy."""
    desc, coeffs, want = frame(31 if not fused else 21)
    rng = np.random.default_rng(7)
    for launch_mb in (None, 0):
        p = context(monkeypatch, fused=fused, launch_mb=launch_mb)
        try:
            for trial in range(3 if launch_mb is None else 1):
                order = rng.permutation(desc.num_groups).tolist()
                decoy(p, desc, 10 + trial, want)
                same(p.decode_frame(desc, coeffs, order=order, stream_output=trial % 2 == 0), want,
                     f"LAUNCH_MB={launch_mb} order {order}")
            order = rng.permutation(desc.num_groups).tolist()
            decoy(p, desc, 20, want)
            same(p.decode_frame(desc, coeffs, order=order, sparse=True, stream_output=True), want,
                 f"LAUNCH_MB={launch_mb} sparse, order {order}")
        finally:
            p.close()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("segs", ["2", "5"])
def test_emulated_epf_fused_row_segments_mixed(emu_lib, monkeypatch, segs):
    """The fused kernel's row segments (work units that re-transform their halo block rows) on frames where engaged
    and skipped blocks mix in every block row -- test_emulated_cuda.py's row-segment test engages every block."""
    monkeypatch.setenv("JXLGPU_FUSED_SEGS", segs)
    p = context(monkeypatch, fused=True)
    try:
        for mask, iters in ((21, 1), (28, 2), (30, 3)):       # 28: EPF 1 + 2, 30: EPF 0 + 1 + 2, no Gaborish
            from oracle import cpu
            desc, coeffs = support.epf_frame(270, 330, seed=mask + int(segs), gab=mask & 1, epf_iters=iters)
            want = cpu.render_frame(desc, coeffs, rcp_mode=0)
            decoy(p, desc, mask, want)
            same(p.decode_frame(desc, coeffs), want, f"chain {mask}, {segs} segments")
    finally:
        p.close()
