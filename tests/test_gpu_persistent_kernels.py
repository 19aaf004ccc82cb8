"""-m gpu: the persistent 8x8 transform kernels at the frame sizes where they run, against the oracle.

idct8_tma_kernel is a software pipeline: every warp walks items warp, warp + nwarps, ... with a 4-entry ring of
work-list records and two staging buffers, each behind its own mbarrier.  Only from a warp's third item on does it
wait on a barrier's second phase and issue bulk copies at the end of an item; the small frames of
test_gpu_parity.py give a warp less than one item.  The steady-state tests here first assert, from the frame's
AcStrategy map and the SM count, that every warp of the launch runs at least six items.

The ordinary-load kernel (idct8_kernel) renders device-resident planes that are not 16-byte aligned; it is reached
here through such planes and through JXLGPU_IDCT8_TMA=0.  Bar everywhere: bit-exact vs oracle/jxl_oracle.c in
exact-reciprocal mode."""
import dataclasses

import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi, pipeline

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("built")]

EIGHT = (0, 2, 12, 13, 1, 3, 14, 15, 16, 17)    # the 8x8-class work lists, in the kernels' order
TAP = abi.STAGE_EXPLICIT | 0                   # planar XYB right after the inverse transforms
MIN_ITEMS_PER_WARP = 6


def tma_coverage(desc, num_sms):
    """(8x8-class items, warps of idct8_tma_kernel) for one launch over the whole frame.  Mirrors launch_idct in
    libjxl_b200/csrc/jxl_b200.cu (px_blocks at line 240, run8's grid at lines 259-260): grid = min(2 * SMs,
    px_blocks / 64 + 1) CTAs of kTma8Warps = 16 warps, px_blocks = 1024 per AC group of the launch; an item is up to
    four varblocks of one list (the kernel's pre[] table)."""
    acs = desc.ac_strategy
    counts = np.bincount(acs[(acs & 1) == 1] >> 1, minlength=27)
    items = int(sum((int(counts[s]) + 3) // 4 for s in EIGHT))
    px_blocks = desc.num_groups * 1024
    grid = min(2 * num_sms, px_blocks // 64 + 1)
    return items, grid * 16


def assert_steady_state(desc):
    import torch
    items, warps = tma_coverage(desc, torch.cuda.get_device_properties(0).multi_processor_count)
    print(f"{desc.xsize}x{desc.ysize}: {items} 8x8-class items, {warps} warps, {items / warps:.2f} items per warp")
    assert items // warps >= MIN_ITEMS_PER_WARP, (items, warps)


def assert_same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, what
    if not np.array_equal(got, want):
        d = np.abs(got.astype(np.float64) - want.astype(np.float64))
        raise AssertionError(f"{what}: {int((d > 0).sum())} of {d.size} samples differ, max |diff| {np.nanmax(d):.3e}")


# ---- frames and oracle images, each made once per module ----
FRAMES = {
    "4k-8x8": lambda: wl.synthetic_frame(3840, 2160, seed=3840, strategies=",".join(map(str, EIGHT))),
    "8k-all27": lambda: wl.synthetic_frame(7680, 4320, seed=7680, epf_iters=1, ac_type=abi.AC_INT32),
    "ragged-all27": lambda: wl.synthetic_frame(1201, 531, seed=1201, epf_iters=1),
}


@pytest.fixture(scope="module")
def cache():
    store = {}
    yield store
    store.clear()


def frame(cache, name, ac_type=None, large=False):
    """(desc, coeffs) of FRAMES[name]; `ac_type` converts the coefficients, `large` sets about 2 % of them (int32)
    to magnitudes up to 2^30."""
    if ("frame", name) not in cache:
        cache[("frame", name)] = FRAMES[name]()
    key = ("frame", name, ac_type, large)
    if key not in cache:
        desc, coeffs = cache[("frame", name)]
        if ac_type is not None and ac_type != desc.ac_type:
            desc = dataclasses.replace(desc, ac_type=ac_type)
            coeffs = coeffs.astype(np.int16 if ac_type == abi.AC_INT16 else np.int32)
        if large:
            assert desc.ac_type == abi.AC_INT32
            rng = np.random.default_rng(0)
            big = rng.integers(-(1 << 30), 1 << 30, coeffs.shape, dtype=np.int64).astype(np.int32)
            coeffs = np.where(rng.random(coeffs.shape) < 0.02, big, coeffs).astype(np.int32)
        cache[key] = (desc, coeffs)
    return cache[key]


def with_mask(desc, mask):
    if mask is None:
        return desc
    return dataclasses.replace(desc, stage_mask=mask, out_format=abi.OUT_PLANAR_F32)


def oracle(cache, name, mask=None, ac_type=None, large=False):
    """The oracle's image of a frame; int16 and int32 planes of the same values share it."""
    key = ("oracle", name, mask, large)
    if key not in cache:
        from oracle import cpu
        desc, coeffs = frame(cache, name, ac_type, large)
        cache[key] = cpu.render_frame(with_mask(desc, mask), coeffs, rcp_mode=0)
    return cache[key]


# ---- contexts and device-resident rendering ----
def context(monkeypatch, fused=False, tma=True, launch_mb=None):
    """A new context: JXLGPU_FUSED / JXLGPU_IDCT8_TMA / JXLGPU_LAUNCH_MB are read when it is created."""
    monkeypatch.setenv("JXLGPU_FUSED", "1" if fused else "0")
    monkeypatch.setenv("JXLGPU_IDCT8_TMA", "1" if tma else "0")
    if launch_mb is None:
        monkeypatch.delenv("JXLGPU_LAUNCH_MB", raising=False)
    else:
        monkeypatch.setenv("JXLGPU_LAUNCH_MB", str(launch_mb))
    return pipeline.TransformPipeline(device=0, num_host_threads=1)


def device_planes(coeffs, offset=None):
    """The three planes in device memory: one tensor (16-byte aligned), or with `offset` each plane in its own
    byte allocation, starting `offset` bytes past a 16-byte boundary.  Returns (tensors to keep, addresses)."""
    import torch
    if offset is None:
        dev = torch.from_numpy(coeffs).cuda()
        return [dev], [dev[c].data_ptr() for c in range(3)]
    keep, ptrs = [], []
    for c in range(3):
        src = torch.from_numpy(np.ascontiguousarray(coeffs[c]).view(np.uint8).reshape(-1))
        raw = torch.empty(src.numel() + 32, dtype=torch.uint8, device="cuda")
        o = (-raw.data_ptr()) % 16 + offset
        raw[o:o + src.numel()].copy_(src)
        keep.append(raw)
        ptrs.append(raw.data_ptr() + o)
    return keep, ptrs


def render_resident(p, desc, coeffs, offset=None):
    """set_device_coefficients + frame_begin + render_device into a device buffer.  Returns (pixels, launches)."""
    import torch
    keep, ptrs = device_planes(coeffs, offset)
    out = torch.full(desc.out_shape(), float("nan"), dtype=torch.float32, device="cuda")
    assert desc.out_dtype == np.float32
    p.set_device_coefficients(ptrs)
    try:
        p.frame_begin(desc)
        before = p.launch_count()
        p.render_device(out.data_ptr(), desc.out_row_bytes, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        launches = p.launch_count() - before
    finally:
        p.set_device_coefficients(None)
    got = out.cpu().numpy()
    del out, keep
    torch.cuda.empty_cache()
    return got, launches


# ---- a. the 8x8 class at steady state, device-resident ----
@pytest.mark.parametrize("ac_type,large,mask", [(abi.AC_INT16, False, TAP), (abi.AC_INT32, False, TAP),
                                                (abi.AC_INT32, True, TAP), (abi.AC_INT16, False, None)],
                         ids=["int16-tap", "int32-tap", "int32-2^30-tap", "int16-full-chain"])
def test_idct8_tma_steady_state(cache, monkeypatch, ac_type, large, mask):
    """3840x2160 of the ten 8x8-class strategies, ~7.7 items per warp at 132 SMs: every warp goes round the record
    ring, waits on both barriers at parity 0, 1, 0 and issues the end-of-item bulk copies several times.  The
    2^30 magnitudes run through the tap only (the filters would not stay finite)."""
    desc, coeffs = frame(cache, "4k-8x8", ac_type, large)
    assert_steady_state(desc)
    want = oracle(cache, "4k-8x8", mask, ac_type, large)
    p = context(monkeypatch)
    try:
        got, launches = render_resident(p, with_mask(desc, mask), coeffs)
    finally:
        p.close()
    assert launches == 6
    if large:
        assert np.isfinite(got).all()
    assert_same(got, want, f"ac_type={ac_type} large={large} mask={mask}")


# ---- b. the benchmarked shape ----
@pytest.mark.parametrize("fused", [False, True], ids=["two-kernel", "fused"])
def test_8k_all_strategies_int32(cache, monkeypatch, fused):
    """7680x4320, all 27 strategies, int32, f32 out, Gaborish + one EPF pass (the chain of the benchmark's 8K d1.0
    frame, which the fused kernel takes: 5 launches instead of 6).  Rendered twice: the work lists are filled by
    atomics, so warps get different items each time, and the pixels must not change."""
    desc, coeffs = frame(cache, "8k-all27")
    assert len(wl.strategy_histogram(desc.ac_strategy)) == 27
    assert_steady_state(desc)
    want = oracle(cache, "8k-all27")
    p = context(monkeypatch, fused=fused)
    try:
        got, launches = render_resident(p, desc, coeffs)
        assert launches == (5 if fused else 6)
        assert_same(got, want, "first render")
        del got
        again, _ = render_resident(p, desc, coeffs)
        assert_same(again, want, "second render")
    finally:
        p.close()


# ---- c. the host-fed path at steady state ----
def test_host_fed_launch_split(cache, monkeypatch):
    """JXLGPU_LAUNCH_MB=4096 transforms the whole 3840x2160 frame in one launch (steady state on the host-fed path);
    =0 launches every AC-group row as soon as it is complete.  Both give the oracle's pixels, and the second really
    splits the frame into more launches."""
    desc, coeffs = frame(cache, "4k-8x8", abi.AC_INT16)
    assert_steady_state(desc)
    desc = with_mask(desc, TAP)
    want = oracle(cache, "4k-8x8", TAP, abi.AC_INT16)
    deltas = {}
    for mb in (4096, 0):
        p = context(monkeypatch, launch_mb=mb)
        try:
            before = p.launch_count()
            got = p.decode_frame(desc, coeffs)
            deltas[mb] = p.launch_count() - before
        finally:
            p.close()
        assert_same(got, want, f"JXLGPU_LAUNCH_MB={mb}")
    assert deltas[0] > deltas[4096], deltas


# ---- d. the ordinary-load kernel, reached both ways ----
@pytest.mark.parametrize("name", ["4k-8x8", "ragged-all27"])
@pytest.mark.parametrize("ac_type,offsets", [(abi.AC_INT16, (2, 8)), (abi.AC_INT32, (4, 8))], ids=["int16", "int32"])
def test_idct8_ordinary_loads(cache, monkeypatch, name, ac_type, offsets):
    """Device-resident planes 2 / 4 / 8 bytes past a 16-byte boundary (idct8_kernel: element loads for the rows of
    the specials), and 16-byte aligned planes on a context created with JXLGPU_IDCT8_TMA=0 (idct8_kernel with vector
    loads).  Same pixels as the oracle."""
    desc, coeffs = frame(cache, name, ac_type)
    desc = with_mask(desc, TAP)
    want = oracle(cache, name, TAP, ac_type)
    p = context(monkeypatch)
    try:
        for off in offsets:
            got, launches = render_resident(p, desc, coeffs, offset=off)
            assert launches == 6
            assert_same(got, want, f"planes at +{off}")
    finally:
        p.close()
    p = context(monkeypatch, tma=False)
    try:
        got, launches = render_resident(p, desc, coeffs)
        assert launches == 6
        assert_same(got, want, "JXLGPU_IDCT8_TMA=0")
    finally:
        p.close()


def test_fused_context_falls_back_for_unaligned_planes(cache, monkeypatch):
    """The fused kernel stages coefficients with bulk copies: a fused context given planes that are not 16-byte
    aligned renders on the two-kernel path (6 launches instead of 5), with the same pixels."""
    desc, coeffs = frame(cache, "ragged-all27")
    want = oracle(cache, "ragged-all27")
    p = context(monkeypatch, fused=True)
    try:
        got, launches = render_resident(p, desc, coeffs)
        assert launches == 5
        assert_same(got, want, "fused kernel, aligned planes")
        got, launches = render_resident(p, desc, coeffs, offset=8)
        assert launches == 6
        assert_same(got, want, "fused context, planes at +8")
    finally:
        p.close()


@pytest.mark.parametrize("ac_type,offset", [(abi.AC_INT16, 1), (abi.AC_INT32, 2)], ids=["int16+1", "int32+2"])
def test_element_misaligned_planes_are_refused(cache, monkeypatch, ac_type, offset):
    """Planes not aligned to the element size cannot be loaded at all: render_device refuses them before it
    launches anything, and the context renders aligned planes afterwards."""
    import torch
    desc, coeffs = frame(cache, "ragged-all27", ac_type)
    desc = with_mask(desc, TAP)
    p = context(monkeypatch)
    try:
        keep, ptrs = device_planes(coeffs, offset)
        out = torch.empty(desc.out_shape(), dtype=torch.float32, device="cuda")
        p.set_device_coefficients(ptrs)
        try:
            p.frame_begin(desc)
            before = p.launch_count()
            with pytest.raises(pipeline.JxlGpuError) as e:
                p.render_device(out.data_ptr(), desc.out_row_bytes, torch.cuda.current_stream().cuda_stream)
            assert e.value.code == abi.ERR_INVALID_ARGUMENT
            assert p.launch_count() == before
        finally:
            p.set_device_coefficients(None)
        del keep, out
        got, _ = render_resident(p, desc, coeffs)
        assert_same(got, oracle(cache, "ragged-all27", TAP, ac_type), "after the refusal")
    finally:
        p.close()
