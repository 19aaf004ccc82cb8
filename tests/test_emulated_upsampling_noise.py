"""Upsampling (4x, 8x) and noise on the CPU emulation of the product's CUDA source (tests/emu), at emulator sizes:
custom F16 weights, a strength LUT that reaches every branch, ragged output sizes, every output format and entry point,
each checked render after a decoy, and the replica refusal.  Bit-exact against the oracle.  The GPU mirror is
tests/test_gpu_upsampling_noise.py.  Wall time on 8 cores: about six minutes (each render of a 4x / 8x frame takes
5-9 s of SIMT emulation)."""
import ctypes as C

import numpy as np
import pytest

import jxl_workload as wl
from libjxl_b200 import abi, pipeline
from tests import support

FORMATS = [(abi.OUT_RGB_F32, 0), (abi.OUT_PLANAR_F32, 0), (abi.OUT_RGB_U8, abi.STAGE_SRGB),
           (abi.OUT_RGBA_U8, abi.STAGE_SRGB), (abi.OUT_RGB_U16, 0), (abi.OUT_RGB_F16, abi.STAGE_SRGB)]
SIZES = {4: (60, 41), 8: (40, 30)}      # outputs 237 x 163 and 313 x 239: ragged 256-tiles, widths not multiples of 16


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu import build_emu
    so = build_emu.build()
    saved = pipeline._lib
    pipeline._lib = pipeline.bind(C.CDLL(str(so)))
    try:
        yield pipeline._lib
    finally:
        pipeline._lib = saved


@pytest.fixture(scope="module")
def emu(emu_lib):
    p = pipeline.TransformPipeline(device=0, num_host_threads=2)
    yield p
    p.close()


def oracle(desc, coeffs):
    from oracle import cpu
    return cpu.render_frame(desc, coeffs, rcp_mode=0)


def same(a, b):
    if a.dtype == np.float16:
        a, b = a.view(np.uint16), b.view(np.uint16)
    return a.shape == b.shape and np.array_equal(a, b)


def after_decoy(p, desc, coeffs, seed, render=None):
    """Render a decoy (ups_decoy) on `p`, then the frame; the decoy must differ from the frame on 99 % of the pixels."""
    render = render or (lambda d, c: p.decode_frame(d, c))
    want = oracle(desc, coeffs)
    d, dc = support.ups_decoy(desc, seed)
    decoy = render(d, dc)
    assert same(decoy, oracle(d, dc))
    # (8-bit outputs: pixels that both saturate to the same corner of the cube coincide, up to 1.5 % of them)
    eight = desc.out_format in (abi.OUT_RGB_U8, abi.OUT_RGBA_U8)
    support.assert_decoy_differs(decoy, want, desc.out_format == abi.OUT_PLANAR_F32, 0.98 if eight else 0.99)
    return render(desc, coeffs), want


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [4, 8])
def test_emulated_coverage_of_the_scenarios(n):
    """The frames of this file reach what they are meant to: window clamp, every LUT branch, ragged tiles."""
    w, h = SIZES[n]
    desc, coeffs = support.ups_noise_frame(n, w, h, seed=n + w)
    support.ups_noise_coverage(desc, coeffs, f"emulator {n}x")
    desc, coeffs = support.ups_noise_frame(1, 70, 50, seed=3)
    support.ups_noise_coverage(desc, coeffs, "emulator noise only")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fmt,srgb", FORMATS)
@pytest.mark.parametrize("n", [4, 8])
def test_emulated_factor_noise_format(emu, n, fmt, srgb):
    """Custom weights, noise, every output format; after a decoy of other content, indices and weights."""
    w, h = SIZES[n]
    desc, coeffs = support.ups_noise_frame(n, w, h, seed=10 * n + fmt, fmt=fmt, srgb=srgb)
    got, want = after_decoy(emu, desc, coeffs, seed=99 + fmt)
    assert same(got, want)


@pytest.mark.timeout(900)
def test_emulated_noise_only_and_upsampling_only(emu):
    desc, coeffs = support.ups_noise_frame(1, 70, 50, seed=4, fmt=abi.OUT_RGB_U16)
    got, want = after_decoy(emu, desc, coeffs, seed=5)
    assert same(got, want)
    desc, coeffs = support.ups_noise_frame(4, 60, 41, seed=6, noise=False)
    got, want = after_decoy(emu, desc, coeffs, seed=7)
    assert same(got, want)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("mask", [abi.STAGE_GAB | abi.STAGE_EPF2 | abi.STAGE_XYB, abi.STAGE_EPF0 | abi.STAGE_XYB])
def test_emulated_generic_tile_kernel(emu, mask):
    """Chains outside the production set: the generic tile kernel writes ups_in."""
    desc, coeffs = support.ups_noise_frame(4, 60, 41, seed=mask)
    desc.stage_mask = abi.STAGE_EXPLICIT | mask
    got, want = after_decoy(emu, desc, coeffs, seed=mask + 1)
    assert same(got, want)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [4, 8])
def test_emulated_entry_points(emu, n):
    """render_device into a padded buffer (padding untouched), shuffled streaming into the caller's buffer, the
    sparse hand-off: each after a decoy."""
    w, h = SIZES[n]
    desc, coeffs = support.ups_noise_frame(n, w, h, seed=40 + n, fmt=abi.OUT_RGB_U8, srgb=abi.STAGE_SRGB)
    row = desc.out_row_bytes
    stride = row + 40
    oh = desc.out_shape()[0]

    def device(d, c):
        buf = np.full((oh, stride), 0x5A, np.uint8)
        dev = np.ascontiguousarray(c)
        emu.set_device_coefficients([dev[k].ctypes.data for k in range(3)])
        try:
            emu.frame_begin(d)
            emu.render_device(buf.ctypes.data, stride)
            emu.synchronize()
        finally:
            emu.set_device_coefficients(None)
        assert (buf[:, row:] == 0x5A).all()
        return buf[:, :row].copy().reshape(d.out_shape())

    got, want = after_decoy(emu, desc, coeffs, seed=1, render=device)
    assert same(got, want)
    order = np.random.default_rng(n).permutation(desc.num_groups).tolist()
    got, _ = after_decoy(emu, desc, coeffs, seed=2,
                         render=lambda d, c: emu.decode_frame(d, c, order=order, stream_output=True))
    assert same(got, want)
    got, _ = after_decoy(emu, desc, coeffs, seed=3, render=lambda d, c: emu.decode_frame(d, c, sparse=True))
    assert same(got, want)


@pytest.mark.timeout(900)
def test_emulated_context_sequence(emu_lib):
    """One context, frames whose upsampling / noise state must be reset or re-sized between them."""
    p = pipeline.TransformPipeline(device=0, num_host_threads=1)
    try:
        seq = [support.ups_noise_frame(8, 40, 30, seed=1),
               support.ups_noise_frame(2, 61, 37, seed=2, noise=False),
               wl.synthetic_frame(70, 50, seed=3, epf_iters=1),
               support.ups_noise_frame(1, 70, 50, seed=4, frame_index=(9, 2)),
               support.ups_noise_frame(4, 60, 41, seed=5),
               support.ups_noise_frame(8, 17, 9, seed=6)]
        for i, (desc, coeffs) in enumerate(seq):
            assert same(p.decode_frame(desc, coeffs), oracle(desc, coeffs)), i
    finally:
        p.close()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", ["ce", "sm", "kernel"])
def test_emulated_replicas_refused(emu_lib, mode, monkeypatch):
    """Upsampled and noisy frames are finished by upsample_kernel, which writes the local buffer only: with output
    replicas (or a multicast address) set, render_device refuses them before enqueuing anything, and the context
    renders the next frame."""
    if mode == "ce":
        monkeypatch.delenv("JXLGPU_GATHER", raising=False)
    else:
        monkeypatch.setenv("JXLGPU_GATHER", mode)
    p = pipeline.TransformPipeline(device=0, num_host_threads=1)
    try:
        for desc, coeffs in (support.ups_noise_frame(4, 60, 41, seed=8, noise=False),
                             support.ups_noise_frame(1, 70, 50, seed=9)):
            nbytes = oracle(desc, coeffs).nbytes
            dev = np.ascontiguousarray(coeffs)
            local = np.full(nbytes + 32, 0xAB, np.uint8)
            reps = [np.full(nbytes + 32, 0xCD, np.uint8) for _ in range(3)]
            base = lambda a: a.ctypes.data + (-a.ctypes.data) % 16     # noqa: E731
            for replicas, mc in (([base(r) for r in reps], 0), ([], base(reps[0]))):
                p.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
                p.frame_begin(desc)
                p.set_output_replicas(replicas, mc)
                before = p.launch_count()
                try:
                    with pytest.raises(pipeline.JxlGpuError) as e:
                        p.render_device(base(local), desc.out_row_bytes)
                    assert e.value.code == abi.ERR_UNSUPPORTED
                finally:
                    p.set_output_replicas([])
                    p.set_device_coefficients(None)
                assert p.launch_count() == before
                assert (local == 0xAB).all() and all((r == 0xCD).all() for r in reps)
            assert same(p.decode_frame(desc, coeffs), oracle(desc, coeffs))
        # replicas of a frame without upsampling or noise still work on the same context
        desc, coeffs = wl.synthetic_frame(64, 40, seed=10, epf_iters=1)
        want = oracle(desc, coeffs).view(np.uint8).ravel()
        dev = np.ascontiguousarray(coeffs)
        local = np.zeros(want.size + 32, np.uint8)
        reps = [np.zeros(want.size + 32, np.uint8) for _ in range(3)]
        p.set_device_coefficients([dev[c].ctypes.data for c in range(3)])
        p.frame_begin(desc)
        p.set_output_replicas([base(r) for r in reps])
        try:
            p.render_device(base(local), desc.out_row_bytes)
            p.synchronize()
        finally:
            p.set_output_replicas([])
            p.set_device_coefficients(None)
        for r in reps + [local]:
            o = base(r) - r.ctypes.data
            assert np.array_equal(r[o:o + want.size], want)
    finally:
        p.close()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [1, 4, 8])
def test_emulated_float64_model(emu, n):
    """The planar XYB output (no colour stage) against support's float64 model of the upsampling, ConvolveNoise and
    AddNoise, fed with the emulated kernels' own pre-upsampling planes and the oracle's generator planes."""
    w, h = SIZES.get(n, (70, 50))
    desc, coeffs = support.ups_noise_frame(n, w, h, seed=70 + n)
    support.check_float64_model(emu, desc, coeffs, f"emulator {n}x")
