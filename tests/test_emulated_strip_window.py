"""The strip filter's Gaborish register window, under the SIMT emulation of tests/emu (no GPU).  In its 8x unrolled
steady steps (every steady step of the EPF0 chains) filter_strip_body keeps the horizontal pair sums h(T), h(M) of
each channel in registers and reads only the new row's h(B) from the ring; the window is filled from the ring where
those steps begin, and the unaligned steady steps around them read the ring as before.

Segments begin on multiples of 8 (band starts are group rows, segment lengths multiples of 8), so a chain enters its
steady steps at one phase rin & 7 in a frame's top segment and another in every later one (chain 17: 3 and 2,
21: 7 and 5, 29: 0 and 7, 31: 4 and 3), which sets how many unaligned steps come before the window is filled.  Both
are covered here for each chain with Gaborish, in edge strips and an interior strip: whole frames (top segments) and
the second band of a two-band render (later segments).  The steady steps end at phase (frame height) & 7, so the
whole frames take eight consecutive heights: the hand-over from the unrolled steps to the trailing unaligned ones
happens at every phase.  Bit-exact against the oracle."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from libjxl_b200 import abi, pipeline, sharding
from tests import support

W = 520              # strips: 2 edge strips and one interior strip for every chain below
CHAINS = (17, 21, 29, 31)


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu import build_emu
    so = build_emu.build()
    saved = pipeline._lib
    pipeline._lib = pipeline.bind(C.CDLL(str(so)))      # the emulated library instead of libjxl_b200.so
    yield
    pipeline._lib = saved


def frame(chain, h, seed):
    """An EPF-engaged frame (so the EPF passes after Gaborish permute their blocks) with the explicit chain, planar
    f32 output, and its oracle image."""
    from oracle import cpu
    desc, coeffs = support.epf_frame(W, h, seed=seed, gab=1, epf_iters=3)
    desc.stage_mask = abi.STAGE_EXPLICIT | chain
    desc.out_format = abi.OUT_PLANAR_F32
    return desc, coeffs, cpu.render_frame(desc, coeffs, rcp_mode=0)


def same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, what
    if not np.array_equal(got, want):
        d = got != want
        rows = np.nonzero(d.any(axis=(0, 2)))[0]
        raise AssertionError(f"{what}: {int(d.sum())} samples differ, rows {rows.min()}..{rows.max()}")


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("chain", CHAINS)
def test_emulated_window_every_exit_phase(emu_lib, chain):
    """Whole frames of eight consecutive heights: steady entry at the top segment's phase, exit at every phase."""
    p = pipeline.TransformPipeline(device=0, num_host_threads=2)
    try:
        for h in range(72, 80):
            desc, coeffs, want = frame(chain, h, seed=chain + h)
            same(p.decode_frame(desc, coeffs), want, f"chain {chain}, {W}x{h}")
    finally:
        p.close()


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("chain", CHAINS)
def test_emulated_window_later_segment(emu_lib, chain):
    """Two bands of one group row each: the second band's segments begin at row 256, the later-segment phase."""
    desc, coeffs, want = frame(chain, 256 + 75, seed=100 + chain)
    p = pipeline.TransformPipeline(device=0, num_host_threads=2)
    try:
        rows = []
        for y0 in (0, 1):
            d = dataclasses.replace(desc, band_y0_groups=y0, band_ny_groups=1)
            p.frame_begin(d)
            for g in sharding.groups_needed(d, y0, 1):
                p.submit_group(g, [coeffs[c, g] for c in range(3)])
            rows.append(p.frame_finish())
        same(np.concatenate(rows, axis=1), want, f"chain {chain}, two bands")
    finally:
        p.close()
