"""idct8_tma_kernel's work claiming under the SIMT emulation of tests/emu (no GPU): the same cases as
tests/test_gpu_transform_schedule.py at emulator sizes.  The emulator reports two SMs, so the 8x8 kernel runs 4 CTAs
of 16 warps whose fixed first chunks cover 256 items; the frames here have more, and its CTAs run one after the
other, so the first CTA claims nearly every later chunk.  Device-resident render_device and host-fed decode_frame,
each after a render of another frame of the same size, bit-exact against the oracle."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi, pipeline, sharding

EIGHT = (0, 2, 12, 13, 1, 3, 14, 15, 16, 17)
CHUNK = 2                 # kTma8Chunk (libjxl_b200/csrc/jxl_kernels.cuh)
WARPS = 2 * 2 * 16        # 2 CTAs per SM x the emulator's 2 SMs x 16 warps


@pytest.fixture(scope="module")
def emu():
    from tests.emu import build_emu
    so = build_emu.build()
    saved = pipeline._lib
    pipeline._lib = pipeline.bind(C.CDLL(str(so)))      # the emulated library instead of libjxl_b200.so
    p = pipeline.TransformPipeline(device=0, num_host_threads=1)
    yield p
    p.close()
    pipeline._lib = saved


def oracle(desc, coeffs):
    from oracle import cpu
    return cpu.render_frame(desc, coeffs, rcp_mode=0)


def items(desc):
    acs = desc.ac_strategy
    counts = np.bincount(acs[(acs & 1) == 1] >> 1, minlength=27)
    return int(sum((int(counts[s]) + 3) // 4 for s in EIGHT)), counts


def same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, what
    if not np.array_equal(got, want):
        d = got != want
        raise AssertionError(f"{what}: {int(d.sum())} of {d.size} samples differ")


def render_device(p, desc, coeffs):
    dev = np.ascontiguousarray(coeffs)                  # "device" memory is host memory here
    out = np.full(desc.out_shape(), np.nan, desc.out_dtype)
    p.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
    try:
        p.frame_begin(desc)
        p.render_device(out.ctypes.data, desc.out_row_bytes)
        p.synchronize()
    finally:
        p.set_device_coefficients(None)
    return out


def check(p, desc, coeffs, what):
    want = oracle(desc, coeffs)
    decoy = wl.synthetic_frame(desc.xsize, desc.ysize, seed=desc.xsize + 1, epf_iters=1)
    p.decode_frame(*decoy)
    same(render_device(p, desc, coeffs), want, f"{what}, render_device")
    p.decode_frame(*decoy)
    same(p.decode_frame(desc, coeffs), want, f"{what}, decode_frame")
    return want


def ragged_frame():
    """8x8-class strategies only, with an item count that is odd and no multiple of the launch's warps."""
    for h in range(264, 200, -8):
        desc, coeffs = wl.synthetic_frame(520, h, seed=h, strategies=",".join(map(str, EIGHT)), epf_iters=1)
        n, _ = items(desc)
        if n % CHUNK and n % WARPS and n > 2 * CHUNK * WARPS:
            return desc, coeffs
    raise AssertionError("no candidate size has a ragged item count")


@pytest.mark.timeout(1800)
def test_emulated_ragged_item_count_and_repeats(emu):
    """The ragged frame, then it and another frame rendered in turn on the one context."""
    a = ragged_frame()
    want_a = check(emu, *a, "ragged item count")
    b = wl.synthetic_frame(a[0].xsize, a[0].ysize, seed=3, strategies=",".join(map(str, EIGHT)), epf_iters=1)
    want_b = oracle(*b)
    for i in range(4):
        same(render_device(emu, *(a, b)[i % 2]), (want_a, want_b)[i % 2], f"render {i}")


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("strategies,w,h", [("4,5,6,7,8,9,10,11,18,19,20", 512, 256), ("0", 520, 264)],
                         ids=["no-8x8", "dct8-only"])
def test_emulated_frames_with_and_without_8x8(emu, strategies, w, h):
    desc, coeffs = wl.synthetic_frame(w, h, seed=len(strategies), strategies=strategies, epf_iters=1)
    n, counts = items(desc)
    assert n == 0 if strategies != "0" else (n > 2 * CHUNK * WARPS and counts[0] == counts.sum()), (n, counts)
    check(emu, desc, coeffs, strategies)


@pytest.mark.timeout(1800)
def test_emulated_bands(emu):
    desc, coeffs = wl.synthetic_frame(520, 800, seed=41, strategies=",".join(map(str, EIGHT)), epf_iters=1)
    want = oracle(desc, coeffs)
    decoy = wl.synthetic_frame(520, 800, seed=42, epf_iters=1)
    rows = []
    for y0, ny in sharding.band_partition(desc.ysize_groups, 2):
        emu.decode_frame(*decoy)
        d = dataclasses.replace(desc, band_y0_groups=y0, band_ny_groups=ny)
        _, nrows = sharding.band_pixel_rows(d, y0, ny)
        dev = np.ascontiguousarray(coeffs)
        out = np.full(d.out_shape(nrows), np.nan, d.out_dtype)
        emu.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
        try:
            emu.frame_begin(d)
            emu.render_device(out.ctypes.data, d.out_row_bytes)
            emu.synchronize()
        finally:
            emu.set_device_coefficients(None)
        rows.append(out)
    same(np.concatenate(rows, axis=0), want, "2 bands")


@pytest.mark.timeout(1800)
def test_emulated_all_strategies(emu):
    desc, coeffs = wl.synthetic_frame(1040, 520, seed=27, gab=1, epf_iters=3)
    assert len(wl.strategy_histogram(desc.ac_strategy)) == 27
    assert items(desc)[0] > 2 * CHUNK * WARPS
    check(emu, desc, coeffs, "all 27 strategies")
