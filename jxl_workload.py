"""Workloads for tests and bench.py: synthetic images, reference-made frames, synthetic frames.

Two kinds of frame inputs:
  * `reference_frame(...)`: a seeded synthetic image is encoded by the reference encoder and
    opened with the reference's own FrameDecoder (oracle/ref_harness.cc), which plays the host
    libjxl here: bitstream -> entropy-decoded coefficient groups + side info.  That hand-off is
    what the C ABI receives in a real integration (INTEGRATION.md); it is workload
    preparation, untimed, and not on the product path.
  * `synthetic_frame(...)`: no reference needed; random coefficients and a strategy map that
    cycles through all 27 AcStrategy types (cjxl never emits > 64x64, SURVEY.md §8c caveat).
"""
from __future__ import annotations

import hashlib
import os
import pickle
from pathlib import Path

import numpy as np

from libjxl_b200 import abi

ROOT = Path(__file__).resolve().parent
CACHE = Path(os.environ.get("JXL_B200_CACHE", "/tmp/jxl_b200_cache"))


def synth_image(w: int, h: int, seed: int = 1234, kind: str = "photo") -> np.ndarray:
    """Seeded RGB8 test image (BASELINE.md §3: low-frequency gradients + 4x4-block noise
    sigma 12 + pixel noise sigma 4 + two hard edges; `noise` = uniform noise)."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = (128 + 60 * np.sin(xx / 37.0)[..., None] * np.array([1, 0.7, 0.4], np.float32)
           + 40 * np.cos(yy / 23.0)[..., None] * np.array([0.3, 1, 0.6], np.float32))
    if kind == "photo":
        blk = rng.normal(0, 12, ((h + 3) // 4, (w + 3) // 4, 3)).astype(np.float32)
        img += np.repeat(np.repeat(blk, 4, 0), 4, 1)[:h, :w]
        img += rng.normal(0, 4, (h, w, 3)).astype(np.float32)
    else:  # "smooth": large transforms dominate
        img += 20 * np.sin((xx + 2 * yy) / 91.0)[..., None]
        img += rng.normal(0, 0.7, (h, w, 3)).astype(np.float32)
    img[h // 5: 2 * h // 5, 3 * w // 5: 4 * w // 5] += 80
    img[3 * h // 5: 4 * h // 5, w // 6: w // 3] -= 70
    return np.clip(img, 0, 255).astype(np.uint8)


def strategy_histogram(ac_strategy: np.ndarray) -> dict[str, int]:
    first = ac_strategy[(ac_strategy & 1) == 1] >> 1
    cnt = np.bincount(first, minlength=27)
    return {abi.STRATEGY_NAMES[i]: int(c) for i, c in enumerate(cnt) if c}


def reference_frame(w: int, h: int, distance: float = 1.0, effort: int = 7, gaborish: int = -1,
                    epf: int = -1, seed: int = 1234, kind: str = "photo", threads: int | None = None,
                    cache: bool = True, want_decoded: bool = True):
    """Returns dict(desc, coeffs, jxl, decoded, hist, bpp). Uses oracle/_ref (the reference)."""
    from oracle import cpu as ocpu
    from oracle import ref
    key = hashlib.sha1(f"v2-{w}x{h}-d{distance}-e{effort}-g{gaborish}-p{epf}-s{seed}-{kind}".encode()).hexdigest()[:16]
    path = CACHE / f"frame_{key}.pkl"
    if cache and path.exists():
        with open(path, "rb") as f:
            out = pickle.load(f)
        out["desc"] = ocpu.desc_from_dump(out.pop("dump"))
        return out
    img = synth_image(w, h, seed, kind)
    threads = threads or os.cpu_count() or 1
    data = ref.encode_rgb8(img, distance, effort, gaborish, epf, threads)
    fr = ref.Frame(data, threads)
    d = fr.dump()
    fr.close()
    out = {"coeffs": d.coeffs, "jxl": data, "decoded": d.decoded if want_decoded else None,
           "hist": strategy_histogram(d.ac_strategy), "bpp": 8.0 * len(data) / (w * h)}
    if cache:
        CACHE.mkdir(parents=True, exist_ok=True)
        dd = _DumpLite(d)
        with open(path, "wb") as f:
            pickle.dump({**out, "dump": dd}, f, protocol=4)
    out["desc"] = ocpu.desc_from_dump(d)
    return out


class _InfoLite:
    pass


class _DumpLite:
    """Picklable copy of oracle.ref.FrameDump (ctypes structs do not pickle)."""

    def __init__(self, d):
        self.info = _InfoLite()
        for name, _ in type(d.info)._fields_:
            v = getattr(d.info, name)
            setattr(self.info, name, list(v) if hasattr(v, "__len__") else v)
        for k in ("ac_strategy", "raw_quant", "sharpness", "ytox", "ytob", "dc", "sigma", "dequant",
                  "dequant_offsets"):
            setattr(self, k, getattr(d, k))


# ---------------------------------------------------------------------------------------------------------------
# Non-default frame-header / image-metadata parameters
# ---------------------------------------------------------------------------------------------------------------
# The scalars of jxlgpu_frame that the frame header (LoopFilter, the DC colour-correlation header, the quantiser's
# qm scales) and the image metadata (OpsinInverseMatrix, intensity target) carry.  `header_params` returns a full
# set of them with legal bitstream values: F16-representable where the header stores F16, |1 + 4 (w1 + w2)| >= 1e-8
# per Gaborish channel, |cfl_base| <= 4, the colour factor from its U32 distribution, x/b_dm = 1.25^-(qm_scale - 2)
# and the opsin matrix scaled by 255 / intensity_target like OpsinParams (InitSIMDInverseMatrix).
HEADER_FIELDS = ("x_dm_multiplier", "b_dm_multiplier", "quant_biases", "cfl_base_x", "cfl_base_b", "cfl_color_scale",
                 "gab_weights", "epf_sharp_lut", "epf_channel_scale", "epf_quant_mul", "epf_pass0_sigma_scale",
                 "epf_pass2_sigma_scale", "epf_border_sad_mul", "inverse_opsin_matrix", "opsin_biases",
                 "opsin_biases_cbrt")
HEADER_SETS = ("pq10000", "dim80", "edges")
# the spec's inverse opsin absorbance matrix (lib/jxl/cms/opsin_params.h), float32 like the reference's constant
SPEC_INVERSE_OPSIN = np.array([[11.031566901960783, -9.866943921568629, -0.16462299647058826],
                               [-3.254147380392157, 4.418770392156863, -0.16462299647058826],
                               [-3.6588512862745097, 2.7129230470588235, 1.9459282392156863]], np.float32)
SPEC_OPSIN_BIAS = -0.0037930732552754493


def f16(v):
    """Round to the nearest binary16 value (what an F16 header field can carry), as float32."""
    return np.asarray(v, np.float64).astype(np.float16).astype(np.float32)


def cbrtf(x: float) -> float:
    """The C library's cbrtf, which OutputEncodingInfo::SetFromMetadata applies to the opsin biases."""
    import ctypes
    import ctypes.util
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.cbrtf.restype, libm.cbrtf.argtypes = ctypes.c_float, [ctypes.c_float]
    return float(libm.cbrtf(float(np.float32(x))))


def _header(gab, lut, epf_scale, epf_quant_mul, pass0, pass2, border, cfl_x, cfl_b, color_factor, x_qm, b_qm,
            quant_biases, inverse_matrix, biases, intensity_target) -> dict:
    gab = f16(gab)
    for c in range(3):
        assert abs(1.0 + 4.0 * (float(gab[2 * c]) + float(gab[2 * c + 1]))) >= 1e-8, gab
    cfl_x, cfl_b = float(f16(cfl_x)), float(f16(cfl_b))
    assert abs(cfl_x) <= 4 and abs(cfl_b) <= 4
    assert 2 <= color_factor < 258 + 65536    # U32: 84 | 256 | 2 + 8 bits | 258 + 16 bits
    assert 0 <= x_qm <= 7 and 0 <= b_qm <= 7
    it = np.float32(f16(intensity_target))
    m = (f16(inverse_matrix).astype(np.float32) * (np.float32(255.0) / it)).astype(np.float32)
    biases = f16(biases)
    return dict(
        x_dm_multiplier=float(np.float32(np.float32(1 / 1.25) ** np.float32(x_qm - 2))),
        b_dm_multiplier=float(np.float32(np.float32(1 / 1.25) ** np.float32(b_qm - 2))),
        quant_biases=tuple(float(v) for v in f16(quant_biases)),
        cfl_base_x=cfl_x, cfl_base_b=cfl_b, color_factor=int(color_factor),
        cfl_color_scale=float(np.float32(1.0) / np.float32(color_factor)),
        gab_weights=tuple(float(v) for v in gab),
        epf_sharp_lut=tuple(float(v) for v in f16(lut)),
        epf_channel_scale=tuple(float(v) for v in f16(epf_scale)),
        epf_quant_mul=float(f16(epf_quant_mul)), epf_pass0_sigma_scale=float(f16(pass0)),
        epf_pass2_sigma_scale=float(f16(pass2)), epf_border_sad_mul=float(f16(border)),
        inverse_opsin_matrix=tuple(float(v) for v in m.ravel()),
        opsin_biases=tuple(float(v) for v in biases), opsin_biases_cbrt=tuple(cbrtf(v) for v in biases),
        intensity_target=float(it))


def header_params(which: str | int) -> dict:
    """A full non-default header: one of HEADER_SETS by name, or a seeded random legal one for an int.
    Every per-channel field differs between channels.  Keys: HEADER_FIELDS + intensity_target, color_factor."""
    custom = SPEC_INVERSE_OPSIN * np.array([[1.03, 0.98, 1.2], [0.96, 1.05, 0.8], [1.02, 0.97, 1.04]], np.float32)
    if which == "pq10000":   # HDR (PQ at 10000 nits), spec matrix, large CfL base, colour factor 256
        return _header(gab=(0.13, 0.047, 0.1, 0.066, 0.125, 0.04), lut=(0, 0.1, 0.3, 0.45, 0.6, 0.8, 1.0, 1.25),
                       epf_scale=(32.0, 6.0, 2.5), epf_quant_mul=0.55, pass0=0.75, pass2=5.0, border=0.75,
                       cfl_x=0.25, cfl_b=0.875, color_factor=256, x_qm=3, b_qm=1,
                       quant_biases=(0.93, 0.95, 0.9, 0.16), inverse_matrix=SPEC_INVERSE_OPSIN,
                       biases=(-0.0035, -0.0041, -0.003), intensity_target=10000)
    if which == "dim80":     # dim display, custom matrix, negative Gaborish weight, colour factor 2..257
        return _header(gab=(-0.0625, 0.11, 0.09, 0.07, 0.16, -0.02), lut=(0.05, 0.2, 0, 0.5, 0.7, 1.1, 0.9, 1.5),
                       epf_scale=(48.0, 4.0, 4.5), epf_quant_mul=0.38, pass0=1.125, pass2=8.0, border=0.5,
                       cfl_x=-0.5, cfl_b=1.5, color_factor=37, x_qm=0, b_qm=5,
                       quant_biases=(0.96, 0.91, 0.94, 0.12), inverse_matrix=custom,
                       biases=(-0.0042, -0.0033, -0.0038), intensity_target=80)
    if which == "edges":     # colour factor beyond 257, negative B base, strongly negative Gaborish channel
        return _header(gab=(0.1, 0.06, -0.15, -0.05, 0.2, 0.1), lut=(1.75, 0, 0.25, 0.125, 0.875, 2.0, 0.625, 1.0),
                       epf_scale=(20.0, 9.0, 1.5), epf_quant_mul=0.7, pass0=0.625, pass2=3.5, border=1.0,
                       cfl_x=1.25, cfl_b=-2.0, color_factor=1000, x_qm=7, b_qm=2,
                       quant_biases=(0.9, 0.97, 0.92, 0.2), inverse_matrix=custom.T.copy(),
                       biases=(-0.0031, -0.0045, -0.0036), intensity_target=255)
    rng = np.random.default_rng(int(which))
    while True:
        gab = rng.uniform(-0.2, 0.3, 6)
        if all(abs(1 + 4 * (gab[2 * c] + gab[2 * c + 1])) >= 0.05 for c in range(3)):
            break
    lut = rng.uniform(0, 1.6, 8)
    if rng.random() < 0.5:
        lut[rng.integers(0, 8)] = 0
    factor = (84, 256, int(rng.integers(2, 258)), int(rng.integers(258, 4000)))[int(rng.integers(0, 4))]
    it = float(rng.choice([80.0, 255.0, 1000.0, 4000.0, 10000.0, float(rng.uniform(50, 10000))]))
    return _header(gab=gab, lut=lut, epf_scale=rng.uniform(1, 60, 3), epf_quant_mul=rng.uniform(0.2, 1.0),
                   pass0=rng.uniform(0.5, 1.5), pass2=rng.uniform(2, 10), border=rng.uniform(0.3, 1.2),
                   cfl_x=rng.uniform(-1.5, 1.5), cfl_b=rng.uniform(-1.5, 2.5), color_factor=factor,
                   x_qm=int(rng.integers(0, 8)), b_qm=int(rng.integers(0, 8)),
                   quant_biases=np.array([0.945, 0.93, 0.95, 0.145]) * rng.uniform(0.85, 1.1, 4),
                   inverse_matrix=SPEC_INVERSE_OPSIN * rng.uniform(0.9, 1.1, (3, 3)).astype(np.float32),
                   biases=SPEC_OPSIN_BIAS * rng.uniform(0.7, 1.3, 3), intensity_target=it)


def apply_header(desc: abi.FrameDesc, hdr: dict) -> abi.FrameDesc:
    """Write the HEADER_FIELDS of `hdr` into `desc` (in place; returns it)."""
    for k in HEADER_FIELDS:
        setattr(desc, k, hdr[k])
    return desc


def synthetic_dequant_table(rng) -> tuple[np.ndarray, np.ndarray]:
    """A smooth, strictly positive stand-in for DequantMatrices (values only need to be
    plausible: parity tests compare the CUDA path and the oracle on the SAME table)."""
    offs = np.zeros((27, 3), np.uint32)
    parts = []
    pos = 0
    for s in range(27):
        r, c = abi.COVERED_Y[s] * 8, abi.COVERED_X[s] * 8
        n = r * c
        lo, hi = min(r, c), max(r, c)
        ky, kx = np.mgrid[0:lo, 0:hi].astype(np.float32)
        rad = np.sqrt((ky / lo) ** 2 + (kx / hi) ** 2)
        for ch in range(3):
            m = (0.00012 + 0.0012 * rad ** 1.5) * (1.0 + 0.1 * ch) * (1 + 0.05 * rng.random((lo, hi), dtype=np.float32))
            offs[s, ch] = pos
            parts.append(m.astype(np.float32).ravel())
            pos += n
    return np.concatenate(parts), offs


def synthetic_frame(w: int, h: int, seed: int = 7, strategies: str = "all", gab: int = 1,
                    epf_iters: int = 3, ac_type: int = abi.AC_INT16, density: float = 0.15):
    """Random frame covering every AcStrategy. Returns (desc, coeffs (3, num_groups, 65536))."""
    rng = np.random.default_rng(seed)
    xb, yb = (w + 7) // 8, (h + 7) // 8
    xg, yg = (xb + 31) // 32, (yb + 31) // 32
    acs = np.zeros((yb, xb), np.uint8)
    filled = np.zeros((yb, xb), bool)
    order = list(range(27)) if strategies == "all" else [int(s) for s in strategies.split(",")]
    # Every group starts with one "primary" multi-block transform at its origin (cycling through
    # all of them, largest first), the rest is filled round-robin with whatever fits, aligned to
    # the transform's own size.
    big_first = sorted(order, key=lambda s: -abi.COVERED_X[s] * abi.COVERED_Y[s])
    multi = [s for s in big_first if abi.COVERED_X[s] * abi.COVERED_Y[s] > 1] or big_first
    pick = 0

    def place(s, x, y):
        cx, cy = abi.COVERED_X[s], abi.COVERED_Y[s]
        acs[y:y + cy, x:x + cx] = s << 1
        acs[y, x] |= 1
        filled[y:y + cy, x:x + cx] = True

    for gy in range(yg):
        for gx in range(xg):
            x0, y0 = gx * 32, gy * 32
            nbx, nby = min(32, xb - x0), min(32, yb - y0)
            for k in range(len(multi)):
                s = multi[(gy * xg + gx + k) % len(multi)]
                if abi.COVERED_X[s] <= nbx and abi.COVERED_Y[s] <= nby:
                    place(s, x0, y0)
                    break
            for by in range(nby):
                for bx in range(nbx):
                    if filled[y0 + by, x0 + bx]:
                        continue
                    for attempt in range(len(order)):
                        s = order[(pick + attempt) % len(order)]
                        cx, cy = abi.COVERED_X[s], abi.COVERED_Y[s]
                        if bx % cx or by % cy or bx + cx > nbx or by + cy > nby:
                            continue
                        if filled[y0 + by:y0 + by + cy, x0 + bx:x0 + bx + cx].any():
                            continue
                        place(s, x0 + bx, y0 + by)
                        pick += 1 + attempt
                        break
                    else:
                        raise AssertionError("no strategy fits")
    first = (acs & 1) == 1
    quant = np.where(first, rng.integers(1, 257, (yb, xb)), 0).astype(np.int32)
    dc = rng.normal(0, 0.08, (3, yb, xb)).astype(np.float32)
    dc[1] += 0.35
    dc[2] += 0.3
    cm = ((yb + 7) // 8, (xb + 7) // 8)
    ytox = rng.integers(-20, 21, cm).astype(np.int8)
    ytob = rng.integers(-20, 21, cm).astype(np.int8)
    sharp = rng.integers(0, 8, (yb, xb)).astype(np.uint8)
    dq, offs = synthetic_dequant_table(rng)
    m, bias, cbrt = abi.default_opsin()
    desc = abi.FrameDesc(
        xsize=w, ysize=h, ac_strategy=acs, raw_quant=quant, dc=dc, ytox=ytox, ytob=ytob, dequant=dq,
        dequant_offsets=offs, inv_global_scale=65536.0 / 24000.0, quant_scale=24000.0 / 65536.0,
        x_dm_multiplier=0.8, b_dm_multiplier=1.25, gab=gab, epf_iters=epf_iters, epf_sharpness=sharp,
        inverse_opsin_matrix=m, opsin_biases=bias, opsin_biases_cbrt=cbrt, ac_type=ac_type)
    dt = np.int16 if ac_type == abi.AC_INT16 else np.int32
    coeffs = np.zeros((3, xg * yg, 65536), dt)
    for g in range(xg * yg):
        n = desc.group_ncoeff(g)
        lap = rng.laplace(0, 2.0, (3, n))
        keep = rng.random((3, n)) < density
        q = np.where(keep, np.rint(lap), 0)
        big = rng.random((3, n)) < 0.002
        q = np.where(big, rng.integers(-300, 301, (3, n)), q)
        coeffs[:, g, :n] = q.astype(dt)
    return desc, coeffs
