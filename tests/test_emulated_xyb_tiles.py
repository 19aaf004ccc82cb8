"""The XYB intermediate in 8x8 block tiles ([3][yb][xb][64], FrameDev::xyb_off), under the SIMT emulation of tests/emu
(no GPU): every producer (8x8 class, mid and large transforms up to 256x256) and every consumer (strip filter, tile
filter, upsampling, the fused kernel's copy blocks) at sizes that are not multiples of 8 or 256, a band whose halo
cuts a large varblock of the next group row, and jxlgpu_device_xyb's row-major copy against the oracle's post-IDCT
planes.  Bit-exact against the oracle."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi, pipeline, sharding


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu import build_emu
    so = build_emu.build()
    saved = pipeline._lib
    pipeline._lib = pipeline.bind(C.CDLL(str(so)))      # the emulated library instead of libjxl_b200.so
    yield
    pipeline._lib = saved


def context(monkeypatch, fused=False):
    monkeypatch.setenv("JXLGPU_FUSED", "1" if fused else "0")
    return pipeline.TransformPipeline(device=0, num_host_threads=2)


def oracle(desc, coeffs):
    from oracle import cpu
    return cpu.render_frame(desc, coeffs, rcp_mode=0)


def device_xyb(pipe, desc):
    ptr, plane_stride, row_stride = pipe.device_xyb()
    assert row_stride == 8 * ((desc.xsize + 7) // 8) and plane_stride == row_stride * 8 * ((desc.ysize + 7) // 8)
    planes = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(3, plane_stride // row_stride, row_stride))
    return planes[:, :desc.ysize, :desc.xsize].copy()


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("w,h,ac_type", [(780, 523, abi.AC_INT16), (263, 91, abi.AC_INT32)])
def test_emulated_tiles_every_producer(emu_lib, monkeypatch, w, h, ac_type):
    """The all-strategy frame (780 x 523 holds all 27 strategies, 128x128 and 256x256 included): post-IDCT planes
    through jxlgpu_device_xyb, the production chain, and the tile kernel."""
    desc, coeffs = wl.synthetic_frame(w, h, seed=w + h, ac_type=ac_type)
    if w == 780:
        assert len(np.unique(desc.ac_strategy >> 1)) == 27
    pipe = context(monkeypatch)
    try:
        assert np.array_equal(pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))          # strip kernel
        tap = dict(stage_mask=abi.STAGE_EXPLICIT, out_format=abi.OUT_PLANAR_F32)
        want = oracle(dataclasses.replace(desc, **tap), coeffs)
        assert np.array_equal(device_xyb(pipe, desc), want)
        desc.stage_mask = abi.STAGE_EXPLICIT | abi.STAGE_GAB | abi.STAGE_EPF1 | abi.STAGE_XYB
        assert np.array_equal(pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))          # tile kernel
    finally:
        pipe.close()


@pytest.mark.timeout(1800)
def test_emulated_tiles_band_cuts_large_varblock(emu_lib, monkeypatch):
    """Two bands of one AC-group row each: the first band's filters read the top rows of the second group row,
    which starts with a 128x256 varblock (DCT128X256); the band renders stitch into the whole frame."""
    desc, coeffs = wl.synthetic_frame(300, 460, seed=3)
    s = desc.ac_strategy >> 1
    assert abi.COVERED_Y[int(s[32, 0])] >= 16
    want = oracle(desc, coeffs)
    pipe = context(monkeypatch)
    try:
        rows = []
        for (y0, ny) in sharding.band_partition(desc.ysize_groups, 2):
            desc.band_y0_groups, desc.band_ny_groups = y0, ny
            pipe.frame_begin(desc)
            for gidx in sharding.groups_needed(desc, y0, ny):
                pipe.submit_group(gidx, [coeffs[c, gidx] for c in range(3)])
            rows.append(pipe.frame_finish())
        assert np.array_equal(np.concatenate(rows, axis=0), want)
    finally:
        pipe.close()


@pytest.mark.timeout(1800)
def test_emulated_tiles_upsampled_frame(emu_lib, monkeypatch):
    """2x upsampling: the strip filter reads the tiles and writes planar XYB for upsample_kernel."""
    from tests.test_emulated_cuda import upsampled_frame
    desc, coeffs = upsampled_frame(2, 121, 67, seed=9)
    pipe = context(monkeypatch)
    try:
        assert np.array_equal(pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))
    finally:
        pipe.close()


@pytest.mark.timeout(1800)
def test_emulated_tiles_fused_copy_blocks(emu_lib, monkeypatch):
    """The fused kernel takes the pixels of varblocks larger than 8x8 from the tiles (its copy blocks)."""
    desc, coeffs = wl.synthetic_frame(270, 141, seed=5)
    pipe = context(monkeypatch, fused=True)
    try:
        assert np.array_equal(pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))
    finally:
        pipe.close()
