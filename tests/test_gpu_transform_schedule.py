"""-m gpu: idct8_tma_kernel's work claiming, against the oracle and the host-fed path.

Warps of the 8x8 kernel take their first two chunks of kTma8Chunk (= 2) items at fixed places and claim every later
chunk from a counter that launch_idct zeroes with the list sizes.  A wrong claim loses or repeats items, so every
case here compares whole images: device-resident render_device and host-fed decode_frame (several transform launches
per frame) against oracle/jxl_oracle.c in exact-reciprocal mode, bit for bit.  Device buffers are never cleared, so
each check follows a render of a different frame of the same size: an item that is skipped keeps that frame's
pixels.  Cases: item counts that divide evenly into neither the launch's warps nor the chunk, frames without any
8x8-class varblock and with nothing else, bands, repeated renders on one context, and an all-27-strategy frame."""
import dataclasses
import functools

import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi, pipeline, sharding
from tests.test_gpu_persistent_kernels import EIGHT, assert_same, render_resident, tma_coverage

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("built")]

CHUNK = 2                                        # kTma8Chunk (libjxl_b200/csrc/jxl_kernels.cuh)
MID = "4,5,6,7,8,9,10,11"                        # DCT16x16 .. DCT16x32: idct_mid_kernel
MID_LARGE = MID + ",18,19,20,21,22,23"           # + 64/128-sided transforms: idct_large_kernel


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def oracle(desc, coeffs):
    from oracle import cpu
    return cpu.render_frame(desc, coeffs, rcp_mode=0)


def ctx():
    return pipeline.TransformPipeline(device=0, num_host_threads=1)


def check(p, desc, coeffs, want, what, decoy):
    """decoy, render_device, decoy, decode_frame: both images must be the oracle's."""
    for how in ("render_device", "decode_frame"):
        d_desc, d_coeffs = decoy
        p.decode_frame(d_desc, d_coeffs)
        if how == "render_device":
            got, launches = render_resident(p, desc, coeffs)
            assert launches == 6, what
        else:
            got = p.decode_frame(desc, coeffs)
        assert_same(got, want, f"{what}, {how}")


@functools.lru_cache(maxsize=1)
def ragged_8x8_frame():
    """A 3840x2160-class frame of the ten 8x8-class strategies whose item count is odd and no multiple of the
    launch's warps, with at least six items per warp (so most items are claimed from the counter)."""
    for dh in range(0, 64, 8):
        desc, coeffs = wl.synthetic_frame(3840 - 8, 2160 - dh, seed=3000 + dh, strategies=",".join(map(str, EIGHT)),
                                          epf_iters=1, ac_type=abi.AC_INT32)
        items, warps = tma_coverage(desc, num_sms())
        if items % CHUNK and items % warps and items >= 6 * warps:
            print(f"{desc.xsize}x{desc.ysize}: {items} items, {warps} warps")
            return desc, coeffs
    raise AssertionError("no candidate size has a ragged item count")


def test_ragged_item_count():
    desc, coeffs = ragged_8x8_frame()
    want = oracle(desc, coeffs)
    decoy = wl.synthetic_frame(desc.xsize, desc.ysize, seed=1, epf_iters=1, ac_type=abi.AC_INT32)
    p = ctx()
    try:
        check(p, desc, coeffs, want, "ragged item count", decoy)
    finally:
        p.close()


@pytest.mark.parametrize("strategies,w,h", [(MID, 1920, 1088), (MID_LARGE, 1920, 1088), ("0", 3840, 2160)],
                         ids=["mid-only", "mid-and-large", "dct8-only"])
def test_frames_with_and_without_8x8(strategies, w, h):
    """No 8x8-class varblock at all (the 8x8 kernel has nothing to claim), and only DCT8x8 (the side kernels have
    nothing) at a size where every warp claims chunks from the counter."""
    desc, coeffs = wl.synthetic_frame(w, h, seed=len(strategies), strategies=strategies, epf_iters=1)
    acs = desc.ac_strategy
    counts = np.bincount(acs[(acs & 1) == 1] >> 1, minlength=27)
    eight = int(counts[list(EIGHT)].sum())
    assert eight == (counts.sum() if strategies == "0" else 0), counts
    if strategies == "0":
        items, warps = tma_coverage(desc, num_sms())
        assert items > 2 * CHUNK * warps, (items, warps)
    want = oracle(desc, coeffs)
    decoy = wl.synthetic_frame(w, h, seed=99, epf_iters=1)
    p = ctx()
    try:
        check(p, desc, coeffs, want, strategies, decoy)
    finally:
        p.close()


@pytest.mark.parametrize("world", [2, 3])
def test_bands(world):
    """Each band of a world-rank partition, device-resident, after a decoy: every band's launch starts from a
    zeroed counter."""
    import torch
    desc, coeffs = ragged_8x8_frame()
    want = oracle(desc, coeffs)
    decoy = wl.synthetic_frame(desc.xsize, desc.ysize, seed=2, ac_type=abi.AC_INT32)
    dev = torch.from_numpy(coeffs).cuda()
    p = ctx()
    rows = []
    try:
        for y0, ny in sharding.band_partition(desc.ysize_groups, world):
            p.decode_frame(*decoy)
            d = dataclasses.replace(desc, band_y0_groups=y0, band_ny_groups=ny)
            _, n = sharding.band_pixel_rows(d, y0, ny)
            out = torch.full(d.out_shape(n), float("nan"), dtype=torch.float32, device="cuda")
            p.set_device_coefficients([dev[c].data_ptr() for c in range(3)])
            try:
                p.frame_begin(d)
                p.render_device(out.data_ptr(), d.out_row_bytes, torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
            finally:
                p.set_device_coefficients(None)
            rows.append(out.cpu().numpy())
    finally:
        p.close()
    assert_same(np.concatenate(rows, axis=0), want, f"{world} bands")


def test_repeated_renders_alternating_frames():
    """Two frames of one size rendered in turn, three times each, on one context: every render_device starts from
    a zeroed counter (one that kept counting would hand out items past the end and leave the other frame's
    pixels)."""
    import torch
    a = ragged_8x8_frame()
    b = wl.synthetic_frame(a[0].xsize, a[0].ysize, seed=7, ac_type=abi.AC_INT32)
    wants = [oracle(*a), oracle(*b)]
    p = ctx()
    try:
        for i in range(6):
            desc, coeffs = (a, b)[i % 2]
            got, _ = render_resident(p, desc, coeffs)
            assert_same(got, wants[i % 2], f"render {i}")
    finally:
        p.close()
    torch.cuda.empty_cache()


def test_all_strategies_4k():
    """bench.py's 4k-all27 frame (all 27 strategies, Gaborish + three EPF passes, int16), twice."""
    desc, coeffs = wl.synthetic_frame(4096, 4096, seed=1234, gab=1, epf_iters=3)
    assert len(wl.strategy_histogram(desc.ac_strategy)) == 27
    want = oracle(desc, coeffs)
    decoy = wl.synthetic_frame(4096, 4096, seed=5, gab=1, epf_iters=3)
    p = ctx()
    try:
        check(p, desc, coeffs, want, "4k-all27", decoy)
        got, _ = render_resident(p, desc, coeffs)
        assert_same(got, want, "4k-all27, render_device again")
    finally:
        p.close()
