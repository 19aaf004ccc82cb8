"""CPU execution of the PRODUCT's CUDA source: tests/emu compiles libjxl_b200/csrc/*.cu(h) for the host
against a SIMT emulation shim (one OS thread per CUDA thread, real barriers) and this file runs the
kernels + the C-ABI host code (scheduler, sparse hand-off, DC stage, output packing) against the oracle --
bit for bit, without a GPU.  It does not replace the -m gpu tests (no real memory system, no PTX); it
lets every round start from kernels whose logic is already known to be right.  Small frames only."""
import ctypes as C

import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi, pipeline
from tests import support


@pytest.fixture(scope="module", params=["two-kernel", "fused"])
def emu_pipe(request):
    """Every test of this file runs twice: through the two-kernel path (plan -> IDCT kernels -> strip filter,
    the default) and through the fused decode kernel (JXLGPU_FUSED=1, read when the context is created)."""
    import os
    from tests.emu import build_emu
    so = build_emu.build()
    saved = pipeline._lib
    pipeline._lib = pipeline.bind(C.CDLL(str(so)))      # the emulated library instead of libjxl_b200.so
    old = os.environ.get("JXLGPU_FUSED")
    os.environ["JXLGPU_FUSED"] = "1" if request.param == "fused" else "0"
    try:
        p = pipeline.TransformPipeline(device=0, num_host_threads=2)
        yield p
        p.close()
    finally:
        pipeline._lib = saved
        if old is None:
            os.environ.pop("JXLGPU_FUSED", None)
        else:
            os.environ["JXLGPU_FUSED"] = old


# The fused decode kernel shares its arithmetic (block8_item, the stage bodies) with the two-kernel path; it is run
# on the tests that exercise what is its own -- tiling, rings, scheduling, bulk copies, output staging -- and skipped
# on the rest (every test twice cost the CPU suite ten minutes of SIMT emulation).
FUSED_TESTS = {"test_emulated_golden_frame", "test_emulated_production_chains", "test_emulated_ragged_sizes",
               "test_emulated_fused_kernel_row_segments", "test_emulated_fused_equals_two_kernel_path",
               "test_emulated_sparse_hand_off"}   # (output formats: inside fused_equals_two_kernel_path)


# ... and these exist for the fused kernel only (the two-kernel context would repeat other tests)
FUSED_ONLY = {"test_emulated_fused_kernel_row_segments", "test_emulated_fused_equals_two_kernel_path"}


@pytest.fixture(autouse=True)
def _fused_subset(request):
    cs = getattr(request.node, "callspec", None)
    if cs is None:
        return
    if cs.params.get("emu_pipe") == "fused" and request.node.originalname not in FUSED_TESTS:
        pytest.skip("fused kernel: covered by the tests of FUSED_TESTS")
    if cs.params.get("emu_pipe") == "two-kernel" and request.node.originalname in FUSED_ONLY:
        pytest.skip("a test of the fused kernel")


def oracle(desc, coeffs):
    from oracle import cpu
    return cpu.render_frame(desc, coeffs, rcp_mode=0)


def same(a, b):
    if a.dtype == np.float16:
        a, b = a.view(np.uint16), b.view(np.uint16)
    return a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.timeout(600)
def test_emulated_golden_frame(emu_pipe):
    """tests/golden/frame_small.npz (real bitstream, Gaborish + EPF 0/1/2): strip kernel chain."""
    desc, coeffs, _ = support.golden_desc()
    assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("w,h,ac_type", [(520, 264, abi.AC_INT16), (300, 200, abi.AC_INT32),
                                         (1024, 520, abi.AC_INT16)])   # the last: all nine 64..256 transforms (sliced passes)
def test_emulated_all_strategy_frame(emu_pipe, w, h, ac_type):
    desc, coeffs = wl.synthetic_frame(w, h, seed=w + h, ac_type=ac_type)
    assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("w,h,smoothing", [(520, 264, 1), (2100, 24, 0), (17, 9, 1)])
def test_emulated_dc_stage(emu_pipe, w, h, smoothing):
    """dc_dequant_kernel + dc_smooth_kernel + the frame_begin plumbing (quantised DC in, two DC groups
    per row at 2100 px) == host-prepared DC planes == the oracle's own DC stage."""
    from tests.test_zz_dc_stage_gpu import with_quant_dc
    desc, coeffs = wl.synthetic_frame(w, h, seed=w + h)
    q, gm, dc = with_quant_dc(desc, smoothing)
    desc.dc = dc
    want = emu_pipe.decode_frame(desc, coeffs)
    assert same(want, oracle(desc, coeffs))
    desc.quant_dc, desc.dc_group_mul, desc.dc_smoothing = q, gm, smoothing
    desc.dc_factors, desc.dc_cfl_factors = support.DC_FACTORS, support.DC_CFL
    desc.dc = None
    assert same(emu_pipe.decode_frame(desc, coeffs), want)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("ac_type", [abi.AC_INT16, abi.AC_INT32])
def test_emulated_sparse_hand_off(emu_pipe, ac_type):
    desc, coeffs = wl.synthetic_frame(264, 264, seed=77 + ac_type, ac_type=ac_type)   # 2 x 2 groups
    if ac_type == abi.AC_INT32:
        coeffs = coeffs.copy()
        rng = np.random.default_rng(2)
        for c in range(3):
            g, k = rng.integers(0, desc.num_groups, 100), rng.integers(64, 4096, 100)
            coeffs[c, g, k] = rng.integers(-300000, 300000, 100)
    want = emu_pipe.decode_frame(desc, coeffs)
    assert same(want, oracle(desc, coeffs))
    order = np.random.default_rng(9).permutation(desc.num_groups).tolist()
    assert same(emu_pipe.decode_frame(desc, coeffs, sparse=True, order=order, stream_output=True), want)
    if ac_type == abi.AC_INT16:   # planes really are re-zeroed: an all-zero frame after one with content
        assert same(emu_pipe.decode_frame(desc, np.zeros_like(coeffs), sparse=True),
                    emu_pipe.decode_frame(desc, np.zeros_like(coeffs)))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("srgb", [0, abi.STAGE_SRGB])
@pytest.mark.parametrize("fmt", [abi.OUT_RGB_F32, abi.OUT_PLANAR_F32, abi.OUT_RGB_U8, abi.OUT_RGBA_U8,
                                 abi.OUT_RGB_U16, abi.OUT_RGB_F16])
def test_emulated_output_stages(emu_pipe, fmt, srgb):
    desc, coeffs = wl.synthetic_frame(201, 131, seed=fmt * 2 + (1 if srgb else 0))
    desc.out_format, desc.stage_mask = fmt, srgb
    assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))          # strip kernel
    desc.stage_mask = abi.STAGE_EXPLICIT | abi.STAGE_GAB | abi.STAGE_EPF2 | abi.STAGE_XYB | srgb
    assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))          # tile kernel


@pytest.mark.timeout(900)
@pytest.mark.parametrize("gab", [0, 1])
@pytest.mark.parametrize("epf_iters", [0, 1, 2, 3])
def test_emulated_production_chains(emu_pipe, gab, epf_iters):
    desc, coeffs = wl.synthetic_frame(277, 300, seed=gab * 10 + epf_iters, gab=gab, epf_iters=epf_iters)
    assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))


@pytest.mark.timeout(900)
def test_emulated_bands_and_shuffled_streaming(emu_pipe):
    from libjxl_b200 import sharding
    desc, coeffs = wl.synthetic_frame(260, 700, seed=21)      # 2 x 3 groups
    want = emu_pipe.decode_frame(desc, coeffs)
    assert same(want, oracle(desc, coeffs))
    order = np.random.default_rng(1).permutation(desc.num_groups).tolist()
    assert same(emu_pipe.decode_frame(desc, coeffs, order=order, stream_output=True), want)
    rows = []
    for (y0, ny) in sharding.band_partition(desc.ysize_groups, 2):
        desc.band_y0_groups, desc.band_ny_groups = y0, ny
        emu_pipe.set_device_coefficients(None)
        emu_pipe.frame_begin(desc)
        for gidx in sharding.groups_needed(desc, y0, ny):
            emu_pipe.submit_group(gidx, [coeffs[c, gidx] for c in range(3)])
        rows.append(emu_pipe.frame_finish())
    desc.band_y0_groups = desc.band_ny_groups = 0
    assert same(np.concatenate(rows, axis=0), want)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("w,h", [(1, 1), (9, 17), (255, 257), (264, 72)])
def test_emulated_ragged_sizes(emu_pipe, w, h):
    desc, coeffs = wl.synthetic_frame(w, h, seed=w * 1000 + h)
    assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind,mode", [("f32", "dense"), ("srgb8", "sparse")])
def test_emulated_cpp_host_example(emu_pipe, tmp_path, kind, mode):
    """examples/host_feed.cc (C++ worker threads, shuffled order, streamed output) linked against the
    emulated library: same bytes as the Python mirror."""
    import os
    import subprocess
    import sys
    from pathlib import Path
    from tests.emu import build_emu
    root = Path(__file__).resolve().parents[1]
    sys.path.insert(0, str(root / "examples"))
    import dump_frame
    (tmp_path / "libjxl_b200.so").symlink_to(build_emu.SO)      # what -ljxl_b200 resolves to in this test
    exe = tmp_path / "host_feed"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", str(root / "include"), str(root / "examples" / "host_feed.cc"),
                           "-L", str(tmp_path), "-ljxl_b200", "-pthread", "-o", str(exe)])
    desc, coeffs = wl.synthetic_frame(300, 300, seed=1877)
    if kind == "srgb8":
        desc.out_format, desc.stage_mask = abi.OUT_RGB_U8, abi.STAGE_SRGB
    dump, raw = tmp_path / "frame.bin", tmp_path / "out.raw"
    dump_frame.write_dump(dump, desc, coeffs)
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp_path))
    out = subprocess.run([str(exe), str(dump), str(raw), "3", mode], env=env, capture_output=True, text=True)
    assert out.returncode == 0, (out.stdout, out.stderr)
    got = np.fromfile(raw, desc.out_dtype).reshape(desc.out_shape())
    assert same(got, emu_pipe.decode_frame(desc, coeffs))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fmt,srgb", [(abi.OUT_RGB_F32, 0), (abi.OUT_RGB_U8, abi.STAGE_SRGB), (abi.OUT_RGB_U16, 0),
                                      (abi.OUT_PLANAR_F32, 0)])
def test_emulated_fused_all_gather_replay(emu_pipe, fmt, srgb):
    """REPL=1 instantiation of the strip kernel: every finished row is replayed into the `replica`
    buffers (peer GPUs' frame slots in production) with 8-byte stores plus byte head/tail pieces.  Odd
    width and packed formats make strips start at arbitrary byte offsets; the replicas must end up
    identical to the local output, and nothing outside the band may be touched."""
    desc, coeffs = wl.synthetic_frame(301, 203, seed=90 + fmt)
    desc.out_format, desc.stage_mask = fmt, srgb
    want = oracle(desc, coeffs)
    dev = np.ascontiguousarray(coeffs)                      # "device" memory is host memory here
    emu_pipe.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
    emu_pipe.frame_begin(desc)
    nbytes = want.nbytes
    guard = 64
    local = np.full(nbytes + 2 * guard, 0xAB, np.uint8)
    reps = [np.full(nbytes + 2 * guard, 0xCD, np.uint8) for _ in range(3)]
    base = lambda a: a.ctypes.data + (-a.ctypes.data) % 8 + 8       # 8-byte aligned, inside the guard
    off = base(local) - local.ctypes.data
    emu_pipe.set_output_replicas([base(r) for r in reps])
    try:
        emu_pipe.render_device(base(local), desc.out_row_bytes)
    finally:
        emu_pipe.set_output_replicas([])
        emu_pipe.set_device_coefficients(None)
    flat = want.view(np.uint8).ravel()
    assert np.array_equal(local[off:off + nbytes], flat)
    for r in reps:
        o = base(r) - r.ctypes.data
        assert np.array_equal(r[o:o + nbytes], flat)
        assert (r[:o] == 0xCD).all() and (r[o + nbytes:] == 0xCD).all()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", ["ce", "sm", "kernel"])
def test_emulated_gather_variants(emu_pipe, mode, monkeypatch):
    """The three ways a band reaches the peers' frame buffers (JXLGPU_GATHER, read when a context is created):
    copy-engine copies per row chunk (default), peer_copy_kernel per row chunk (`sm`, 16-byte stores), the replay
    inside the filter kernel (`kernel`).  Same bytes everywhere, nothing outside the band."""
    if mode != "ce":
        monkeypatch.setenv("JXLGPU_GATHER", mode)
    else:
        monkeypatch.delenv("JXLGPU_GATHER", raising=False)
    p = pipeline.TransformPipeline(device=0, num_host_threads=1)
    try:
        for fmt, srgb in ((abi.OUT_RGB_U8, abi.STAGE_SRGB), (abi.OUT_PLANAR_F32, 0)):
            desc, coeffs = wl.synthetic_frame(304, 520, seed=70 + fmt, epf_iters=1)   # three row chunks
            desc.out_format, desc.stage_mask = fmt, srgb
            want = oracle(desc, coeffs).view(np.uint8).ravel()
            dev = np.ascontiguousarray(coeffs)
            p.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
            p.frame_begin(desc)
            guard = 64
            local = np.full(want.size + 2 * guard, 0xAB, np.uint8)
            reps = [np.full(want.size + 2 * guard, 0xCD, np.uint8) for _ in range(3)]
            base = lambda a: a.ctypes.data + (-a.ctypes.data) % 16 + 16
            p.set_output_replicas([base(r) for r in reps])
            try:
                p.render_device(base(local), desc.out_row_bytes)
                p.synchronize()
            finally:
                p.set_output_replicas([])
                p.set_device_coefficients(None)
            off = base(local) - local.ctypes.data
            assert np.array_equal(local[off:off + want.size], want), (mode, fmt)
            for r in reps:
                o = base(r) - r.ctypes.data
                assert np.array_equal(r[o:o + want.size], want), (mode, fmt)
                assert (r[:o] == 0xCD).all() and (r[o + want.size:] == 0xCD).all()
    finally:
        p.close()


@pytest.mark.timeout(900)
def test_emulated_multicast_replay_and_its_limits(emu_pipe):
    """The multimem.st variant of the replay (emulated as a plain store to the one multicast address):
    4-byte granules for the f32 layouts; packed layouts are refused."""
    desc, coeffs = wl.synthetic_frame(203, 131, seed=123)
    want = oracle(desc, coeffs)
    dev = np.ascontiguousarray(coeffs)
    emu_pipe.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
    emu_pipe.frame_begin(desc)
    local, mc = np.zeros(want.nbytes + 16, np.uint8), np.zeros(want.nbytes + 16, np.uint8)
    base = lambda a: a.ctypes.data + (-a.ctypes.data) % 8
    emu_pipe.set_output_replicas([], base(mc))
    try:
        emu_pipe.render_device(base(local), desc.out_row_bytes)
        o = base(mc) - mc.ctypes.data
        assert np.array_equal(mc[o:o + want.nbytes], want.view(np.uint8).ravel())
        desc.out_format = abi.OUT_RGB_U8
        emu_pipe.frame_begin(desc)
        with pytest.raises(pipeline.JxlGpuError):
            emu_pipe.render_device(base(local), desc.out_row_bytes)
    finally:
        emu_pipe.set_output_replicas([])
        emu_pipe.set_device_coefficients(None)


@pytest.mark.timeout(900)
def test_emulated_strided_outputs_and_accessors(emu_pipe):
    """Row strides larger than a dense row (host: cudaMemcpy2D path of frame_finish / streamed output;
    device: render_device into a padded buffer), the context-owned output + XYB accessors, profiling."""
    from oracle import cpu
    desc, coeffs = wl.synthetic_frame(203, 300, seed=31)        # 1 x 2 groups
    want = oracle(desc, coeffs)
    lib = pipeline.lib()
    row = desc.out_row_bytes
    stride = row + 40
    # (a) frame_finish into a strided host buffer
    buf = np.full((desc.ysize, stride), 0x5A, np.uint8)
    emu_pipe.set_device_coefficients(None)
    emu_pipe.frame_begin(desc)
    for g in range(desc.num_groups):
        emu_pipe.submit_group(g, [coeffs[c, g] for c in range(3)])
    assert lib.jxlgpu_frame_finish(emu_pipe._h, buf.ctypes.data, stride) == 0
    assert np.array_equal(buf[:, :row].copy().view(np.float32).reshape(want.shape), want)
    assert (buf[:, row:] == 0x5A).all()
    # (b) streamed output (frame_set_output) with the same stride
    buf[:] = 0x5A
    emu_pipe.frame_begin(desc)
    assert lib.jxlgpu_frame_set_output(emu_pipe._h, buf.ctypes.data, stride) == 0
    for g in reversed(range(desc.num_groups)):
        emu_pipe.submit_group(g, [coeffs[c, g] for c in range(3)])
    assert lib.jxlgpu_frame_finish(emu_pipe._h, buf.ctypes.data, stride) == 0
    assert np.array_equal(buf[:, :row].copy().view(np.float32).reshape(want.shape), want)
    assert (buf[:, row:] == 0x5A).all()
    # (c) render_device into a padded "device" buffer, then the context-owned output and the XYB planes
    dev = np.ascontiguousarray(coeffs)
    emu_pipe.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
    emu_pipe.frame_begin(desc)
    pad = np.full((desc.ysize, stride // 4 + 2), np.float32(-7), np.float32)
    emu_pipe.set_profiling(True)
    emu_pipe.render_device(pad.ctypes.data, pad.shape[1] * 4)
    assert set(emu_pipe.kernel_times_ms()) == {"plan", "idct8", "idct_mid", "idct_large", "filter"}
    emu_pipe.set_profiling(False)
    assert np.array_equal(pad[:, :desc.xsize * 3].reshape(want.shape), want) and (pad[:, desc.xsize * 3:] == -7).all()
    emu_pipe.render_device()                                     # into the context's own buffer
    ptr, s = emu_pipe.device_output()
    own = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(desc.ysize, s // 4))
    assert s == row and np.array_equal(own.reshape(want.shape), want)
    xyb_ptr, plane_stride, row_stride = emu_pipe.device_xyb()
    planes = np.ctypeslib.as_array(C.cast(xyb_ptr, C.POINTER(C.c_float)), shape=(3, plane_stride // row_stride, row_stride))
    desc.stage_mask, desc.out_format = abi.STAGE_EXPLICIT, abi.OUT_PLANAR_F32     # tap: after the inverse transforms
    assert np.array_equal(planes[:, :desc.ysize, :desc.xsize], cpu.render_frame(desc, coeffs, rcp_mode=0))
    emu_pipe.set_device_coefficients(None)


@pytest.mark.timeout(900)
def test_emulated_argument_validation(emu_pipe):
    """Every documented rejection of frame_begin / submit / render, without side effects on the context."""
    lib = pipeline.lib()
    desc, coeffs = wl.synthetic_frame(300, 200, seed=3)

    def begin_rc(mutate):
        s = desc.to_struct()
        mutate(s)
        return lib.jxlgpu_frame_begin(emu_pipe._h, C.byref(s))

    assert begin_rc(lambda s: None) == abi.OK
    assert begin_rc(lambda s: setattr(s, "xsize", 0)) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: setattr(s, "xsize_blocks", s.xsize_blocks + 1)) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: setattr(s, "raw_quant", None)) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: setattr(s, "out_format", 6)) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: setattr(s, "ac_type", 2)) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: s.dequant_offsets.__setitem__(5, s.dequant_offsets[5] + 2)) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: s.dequant_offsets.__setitem__(5, s.dequant_table_floats)) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: (setattr(s, "band_y0_groups", 1), setattr(s, "band_ny_groups", 1))) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: setattr(s, "epf_sharpness", None)) == abi.ERR_INVALID_ARGUMENT   # epf_iters = 3
    assert begin_rc(lambda s: s.dc.__setitem__(1, None)) == abi.ERR_INVALID_ARGUMENT
    # upsampling: factor 2/4/8 only, weights required, upsampled size consistent with the coded size; noise and
    # upsampling are whole-frame features (no band)
    w2 = np.zeros(15, np.float32)
    assert begin_rc(lambda s: setattr(s, "upsampling", 3)) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: setattr(s, "upsampling", 2)) == abi.ERR_INVALID_ARGUMENT          # no weights
    assert begin_rc(lambda s: (setattr(s, "upsampling", 2), setattr(s, "upsampling_weights", w2.ctypes.data),
                               setattr(s, "xsize_upsampled", 2 * s.xsize + 1))) == abi.ERR_INVALID_ARGUMENT
    assert begin_rc(lambda s: (setattr(s, "upsampling", 2), setattr(s, "upsampling_weights", w2.ctypes.data))) == abi.OK
    assert begin_rc(lambda s: (setattr(s, "noise", 1), setattr(s, "band_ny_groups", 1))) == abi.ERR_UNSUPPORTED
    assert begin_rc(lambda s: None) == abi.OK
    # submit: thread id beyond num_host_threads, null channel pointer, too many coefficients
    ptrs = (C.c_void_p * 3)(*[coeffs[c, 0].ctypes.data for c in range(3)])
    assert lib.jxlgpu_submit_group(emu_pipe._h, 0, 2, ptrs, 1000) == abi.ERR_INVALID_ARGUMENT
    assert lib.jxlgpu_submit_group(emu_pipe._h, 0, 0, ptrs, 65537) == abi.ERR_INVALID_ARGUMENT
    bad = (C.c_void_p * 3)(ptrs[0], None, ptrs[2])
    assert lib.jxlgpu_submit_group(emu_pipe._h, 0, 0, bad, 1000) == abi.ERR_INVALID_ARGUMENT
    # output stride smaller than a row, more replicas than the ABI carries
    out = np.zeros((desc.ysize, desc.xsize, 3), np.float32)
    assert lib.jxlgpu_frame_set_output(emu_pipe._h, out.ctypes.data, desc.out_row_bytes - 4) == abi.ERR_INVALID_ARGUMENT
    assert lib.jxlgpu_set_output_replicas(emu_pipe._h, 9, (C.c_void_p * 9)(), None) == abi.ERR_INVALID_ARGUMENT
    assert lib.jxlgpu_set_output_replicas(emu_pipe._h, 1, (C.c_void_p * 1)(out.ctypes.data + 4), None) == abi.ERR_INVALID_ARGUMENT
    # the frame is still usable
    got = emu_pipe.decode_frame(desc, coeffs)
    assert same(got, oracle(desc, coeffs))
    # calls outside a frame
    assert lib.jxlgpu_frame_finish(emu_pipe._h, None, 0) == abi.ERR_STATE
    assert lib.jxlgpu_submit_group(emu_pipe._h, 0, 0, ptrs, 1000) == abi.ERR_STATE


def planes_at_offset(coeffs, offset):
    """The three coefficient planes, each in its own byte buffer starting `offset` bytes past a 16-byte boundary
    (what a caller's sub-allocation can hand to jxlgpu_set_device_coefficients).  Returns (buffers, addresses)."""
    bufs, ptrs = [], []
    for c in range(3):
        src = np.ascontiguousarray(coeffs[c]).view(np.uint8).ravel()
        buf = np.zeros(src.size + 32, np.uint8)
        o = (-buf.ctypes.data) % 16 + offset
        buf[o:o + src.size] = src
        bufs.append(buf)
        ptrs.append(buf.ctypes.data + o)
    return bufs, ptrs


@pytest.mark.timeout(900)
def test_emulated_unaligned_device_planes(emu_pipe):
    """Device-resident planes that are element-aligned but not 16-byte aligned go to idct8_kernel (the bulk copies of
    idct8_tma_kernel need 16 bytes); it must load them without one vector load at a misaligned address (the shim
    counts what the GPU would fault on) and give the oracle's pixels.  Planes that are not even element-aligned are
    refused before anything is launched."""
    lib = pipeline.lib()
    lib.emu_misaligned_loads.restype, lib.emu_misaligned_loads.argtypes = C.c_uint64, [C.c_int]
    frames = [wl.synthetic_frame(96, 64, seed=5, strategies="0,1,2,3,12,13,14,15,16,17"),   # the 8x8 class only
              wl.synthetic_frame(264, 136, seed=6)]                                         # all strategies
    for ac_type, offsets in ((abi.AC_INT16, (2, 8)), (abi.AC_INT32, (4, 8))):
        for desc, coeffs in frames:
            desc.ac_type = ac_type
            coeffs = coeffs.astype(np.int16 if ac_type == abi.AC_INT16 else np.int32)
            desc.stage_mask, desc.out_format = abi.STAGE_EXPLICIT | 0, abi.OUT_PLANAR_F32   # after the transforms
            want = oracle(desc, coeffs)
            for off in offsets:
                bufs, ptrs = planes_at_offset(coeffs, off)
                out = np.full(desc.out_shape(), np.nan, np.float32)
                emu_pipe.set_device_coefficients(ptrs)
                try:
                    emu_pipe.frame_begin(desc)
                    lib.emu_misaligned_loads(1)
                    emu_pipe.render_device(out.ctypes.data, desc.out_row_bytes)
                    misaligned = lib.emu_misaligned_loads(0)
                finally:
                    emu_pipe.set_device_coefficients(None)
                assert misaligned == 0, (desc.xsize, ac_type, off, misaligned)
                assert same(out, want), (desc.xsize, ac_type, off)
    desc, coeffs = frames[0]                       # (int32 after the loop) at +2: not a multiple of 4 bytes
    assert desc.ac_type == abi.AC_INT32
    bufs, ptrs = planes_at_offset(coeffs.astype(np.int32), 2)
    out = np.zeros(desc.out_shape(), np.float32)
    emu_pipe.set_device_coefficients(ptrs)
    try:
        emu_pipe.frame_begin(desc)
        before = emu_pipe.launch_count()
        with pytest.raises(pipeline.JxlGpuError):
            emu_pipe.render_device(out.ctypes.data, desc.out_row_bytes)
        assert lib.jxlgpu_frame_finish(emu_pipe._h, None, 0) == abi.ERR_INVALID_ARGUMENT   # the host-side finish too
        assert emu_pipe.launch_count() == before
    finally:
        emu_pipe.set_device_coefficients(None)


def epf_engaged_frame(w, h, seed, gab=1, epf_iters=3):
    """A synthetic frame whose EPF weights are non-zero (raw_quant 1, sharpness 7 puts sigma above
    kMinSigma; smooth, small coefficients keep the SADs small).  synthetic_frame's random quantisers
    make the EPF a pass-through, which hides filter bugs on tiny images."""
    desc, coeffs = wl.synthetic_frame(w, h, seed=seed, gab=gab, epf_iters=epf_iters, density=0.05)
    desc.raw_quant = np.where(desc.raw_quant > 0, 1, 0).astype(np.int32)
    desc.epf_sharpness = np.full_like(desc.epf_sharpness, 7)
    coeffs = np.clip(coeffs, -2, 2)
    return desc, coeffs


@pytest.mark.timeout(900)
@pytest.mark.parametrize("w,h", [(40, 1), (40, 2), (300, 2), (1, 1), (9, 3), (270, 5)])
@pytest.mark.parametrize("epf_iters", [1, 2, 3])
def test_emulated_tiny_heights_with_epf_engaged(emu_pipe, w, h, epf_iters):
    """Images lower than a stage's border: the vertical mirror must reflect repeatedly like
    Mirror() (lib/jxl/image_ops.h:184-196)."""
    desc, coeffs = epf_engaged_frame(w, h, seed=w * 7 + h, epf_iters=epf_iters)
    want = oracle(desc, coeffs)
    desc2, _ = epf_engaged_frame(w, h, seed=w * 7 + h, epf_iters=0)
    if w * h > 1:   # the filters really change the picture (the test means something)
        assert not np.array_equal(want, oracle(desc2, coeffs))
    assert same(emu_pipe.decode_frame(desc, coeffs), want)


def epf_mixed_frame(w, h, seed, gab=1, epf_iters=3, engaged=0.3):
    """EPF engaged on a random subset of the blocks (sharpness 7 there, 0 elsewhere -- what the reference
    encoder's sharpness map looks like): the strip kernel runs its EPF passes on a block permutation,
    engaged blocks first, and this frame mixes both kinds inside every strip and block row."""
    desc, coeffs = epf_engaged_frame(w, h, seed, gab=gab, epf_iters=epf_iters)
    rng = np.random.default_rng(seed + 99)
    desc.epf_sharpness = np.where(rng.random(desc.epf_sharpness.shape) < engaged, 7, 0).astype(np.uint8)
    return desc, coeffs


@pytest.mark.timeout(900)
@pytest.mark.parametrize("gab", [0, 1])
@pytest.mark.parametrize("epf_iters", [1, 2, 3])
@pytest.mark.parametrize("w,h,engaged", [(523, 90, 0.3), (250, 41, 0.7), (8, 200, 0.5)])
def test_emulated_epf_block_permutation(emu_pipe, w, h, engaged, gab, epf_iters):
    desc, coeffs = epf_mixed_frame(w, h, seed=w + 3 * h + gab, gab=gab, epf_iters=epf_iters, engaged=engaged)
    want = oracle(desc, coeffs)
    desc0, _ = epf_mixed_frame(w, h, seed=w + 3 * h + gab, gab=gab, epf_iters=0, engaged=engaged)
    assert not np.array_equal(want, oracle(desc0, coeffs))
    assert same(emu_pipe.decode_frame(desc, coeffs), want)


@pytest.mark.timeout(900)
def test_emulated_sparse_small_then_large_frame_on_one_context(emu_pipe):
    """The sparse staging buffer must grow when a context is reused for a larger frame."""
    small, cs = wl.synthetic_frame(64, 64, seed=5)
    assert same(emu_pipe.decode_frame(small, cs, sparse=True), oracle(small, cs))
    big, cb = wl.synthetic_frame(1024, 512, seed=6, density=0.9)
    assert same(emu_pipe.decode_frame(big, cb, sparse=True), oracle(big, cb))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("segs", ["2", "5"])
def test_emulated_fused_kernel_row_segments(emu_pipe, segs, monkeypatch):
    """The fused kernel cuts a strip into row segments (work units); each segment re-transforms the block
    rows of its halo.  Segment boundaries must not show in the pixels."""
    monkeypatch.setenv("JXLGPU_FUSED_SEGS", segs)
    for gab, epf_iters in [(1, 1), (1, 2), (0, 3)]:
        desc, coeffs = epf_engaged_frame(270, 330, seed=31 + epf_iters, gab=gab, epf_iters=epf_iters)
        assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))


@pytest.mark.timeout(900)
def test_emulated_fused_equals_two_kernel_path(emu_pipe, monkeypatch):
    """JXLGPU_FUSED=0 (read at context creation) selects the two-kernel path: both give the oracle's pixels,
    in every output format the fused kernel stages through shared memory."""
    from tests.emu import build_emu
    desc, coeffs = wl.synthetic_frame(500, 60, seed=3, gab=1, epf_iters=1, ac_type=abi.AC_INT32)
    monkeypatch.setenv("JXLGPU_FUSED", "1")    # (the fixture's context is one of the two; this one is the fused kernel)
    two = pipeline.TransformPipeline(device=0, num_host_threads=1)
    try:
        for fmt in (abi.OUT_RGB_F32, abi.OUT_PLANAR_F32, abi.OUT_RGBA_U8, abi.OUT_RGB_F16):
            desc.out_format, desc.stage_mask = fmt, abi.STAGE_SRGB if fmt != abi.OUT_RGB_F32 else 0
            a, b = emu_pipe.decode_frame(desc, coeffs), two.decode_frame(desc, coeffs)
            assert same(a, b) and same(a, oracle(desc, coeffs))
    finally:
        two.close()


def upsampled_frame(n, w, h, seed, fmt=abi.OUT_RGB_F32, srgb=0, ragged=True):
    """A synthetic frame whose frame header asks for N-times upsampling (default weights of the codestream,
    tests/golden/upsampling_weights.npz); the image size is not a multiple of N when `ragged`."""
    from pathlib import Path
    wts = np.load(Path(__file__).parent / "golden" / "upsampling_weights.npz")
    desc, coeffs = wl.synthetic_frame(w, h, seed=seed, epf_iters=1)
    desc.upsampling, desc.upsampling_weights = n, wts[f"weights{n}"]
    desc.xsize_upsampled, desc.ysize_upsampled = (n * w - (n - 1), n * h - 1) if ragged else (n * w, n * h)
    desc.out_format, desc.stage_mask = fmt, srgb
    return desc, coeffs


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n,w,h", [(2, 121, 67), (4, 60, 41), (8, 40, 30)])
@pytest.mark.parametrize("fmt,srgb", [(abi.OUT_RGB_F32, 0), (abi.OUT_RGB_U8, abi.STAGE_SRGB), (abi.OUT_PLANAR_F32, 0)])
def test_emulated_upsampling(emu_pipe, n, w, h, fmt, srgb):
    """SURVEY.md §8f rank 4: UpsamplingStage 2x / 4x / 8x after the filters, fused with XYB -> RGB and the
    output packing (upsample_kernel), host-fed and device-resident entry points."""
    desc, coeffs = upsampled_frame(n, w, h, seed=5 + n, fmt=fmt, srgb=srgb)
    want = oracle(desc, coeffs)
    assert want.shape == desc.out_shape(desc.ysize)
    assert same(emu_pipe.decode_frame(desc, coeffs), want)
    desc.band_y0_groups, desc.band_ny_groups = 0, 1       # bands and upsampling do not combine (yet)
    with pytest.raises(pipeline.JxlGpuError):
        emu_pipe.frame_begin(desc)


NOISE_LUT = (0.001, 0.0068, 0.0039, 0.0049, 0.0059, 0.0078, 0.0088, 0.0107)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n,w,h", [(1, 301, 260), (2, 140, 131), (1, 17, 9)])
@pytest.mark.parametrize("fmt,srgb", [(abi.OUT_RGB_F32, 0), (abi.OUT_RGB_U8, abi.STAGE_SRGB)])
def test_emulated_noise(emu_pipe, n, w, h, fmt, srgb):
    """SURVEY.md §8f rank 4: the noise generator (Xorshift128Plus per 256x256 output tile, noise_gen_kernel), the
    convolution and AddNoise fused with XYB -> RGB and the packing (finish_px), alone and behind the upsampling."""
    if n > 1:
        desc, coeffs = upsampled_frame(n, w, h, seed=5 + n, fmt=fmt, srgb=srgb)
    else:
        desc, coeffs = wl.synthetic_frame(w, h, seed=5 + n, epf_iters=1)
        desc.out_format, desc.stage_mask = fmt, srgb
    desc.noise, desc.noise_lut = 1, NOISE_LUT
    desc.visible_frame_index, desc.nonvisible_frame_index = 3, 1
    want = oracle(desc, coeffs)
    assert same(emu_pipe.decode_frame(desc, coeffs), want)
    desc.noise = 0
    assert not same(oracle(desc, coeffs), want)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fmt", [abi.OUT_RGB_F32, abi.OUT_RGB_U8])
@pytest.mark.parametrize("w,h,filters", [(301, 260, 0), (301, 260, 1), (17, 9, 0)])
def test_emulated_ycbcr_colour_transform(emu_pipe, w, h, filters, fmt):
    """JPEG-origin frames (frame_header.color_transform = YCbCr, 4:4:4): kYCbCrStage in the place of the opsin inverse,
    in the strip kernel's epilogue and in the tile kernel."""
    desc, coeffs = wl.synthetic_frame(w, h, seed=5, gab=filters, epf_iters=filters, strategies="0")
    desc.color_transform, desc.out_format = 1, fmt
    assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))
    desc.stage_mask = abi.STAGE_EXPLICIT | abi.STAGE_EPF2 | abi.STAGE_XYB     # tile kernel
    if filters:
        assert same(emu_pipe.decode_frame(desc, coeffs), oracle(desc, coeffs))
