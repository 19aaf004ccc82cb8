"""ctypes binding of oracle/libjxl_oracle.so (the plain-C restatement of the reference
hot path).  TEST INFRASTRUCTURE ONLY -- see oracle/jxl_oracle.c.  Never imported by the
product package.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from libjxl_b200 import abi

HERE = Path(__file__).resolve().parent
SO = HERE / "libjxl_oracle.so"
_lib = None


def build() -> None:
    subprocess.check_call(["make", "-C", str(HERE), "-s"])


def lib():
    global _lib
    if _lib is None:
        if not SO.exists():
            build()
        L = C.CDLL(str(SO))
        L.jxo_transform_to_pixels.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]
        L.jxo_llf_from_dc.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
        L.jxo_scaled_dct.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
        L.jxo_adjust_quant_bias.restype = C.c_float
        L.jxo_adjust_quant_bias.argtypes = [C.c_int, C.c_int32, C.c_void_p, C.c_int]
        L.jxo_compute_sigma.argtypes = [C.POINTER(abi.JxlGpuFrame), C.c_void_p]
        L.jxo_render_frame.argtypes = [C.POINTER(abi.JxlGpuFrame), C.c_void_p * 3, C.c_int, C.c_void_p]
        L.jxo_dequant_dc.restype = None
        L.jxo_dequant_dc.argtypes = [C.c_void_p * 3, C.c_size_t, C.c_size_t, C.c_float * 3, C.c_float,
                                     C.c_float * 3, C.c_void_p]
        L.jxo_adaptive_dc_smoothing.argtypes = [C.c_float * 3, C.c_void_p, C.c_size_t, C.c_size_t]
        L.jxo_srgb_from_linear.restype = C.c_float
        L.jxo_srgb_from_linear.argtypes = [C.c_float]
        L.jxo_make_unsigned.restype = C.c_uint32
        L.jxo_make_unsigned.argtypes = [C.c_float, C.c_int, C.c_size_t, C.c_size_t, C.c_int]
        L.jxo_f16_from_f32.restype = C.c_uint16
        L.jxo_f16_from_f32.argtypes = [C.c_float]
        L.jxo_noise_planes.restype = None
        L.jxo_noise_planes.argtypes = [C.c_uint32, C.c_uint32, C.c_size_t, C.c_size_t, C.c_void_p]
        _lib = L
    return _lib


def transform_to_pixels(strategy: int, coeffs: np.ndarray) -> np.ndarray:
    rows, cols = abi.COVERED_Y[strategy] * 8, abi.COVERED_X[strategy] * 8
    co = np.ascontiguousarray(coeffs, np.float32).ravel()
    assert co.size == rows * cols
    px = np.zeros((rows, cols), np.float32)
    rc = lib().jxo_transform_to_pixels(strategy, co.ctypes.data, px.ctypes.data, cols)
    assert rc == 0
    return px


def llf_from_dc(strategy: int, dc: np.ndarray, block: np.ndarray) -> np.ndarray:
    dc = np.ascontiguousarray(dc, np.float32)
    blk = np.ascontiguousarray(block, np.float32).ravel().copy()
    rc = lib().jxo_llf_from_dc(strategy, dc.ctypes.data, dc.shape[1], blk.ctypes.data)
    assert rc == 0
    return blk


def scaled_dct(pixels: np.ndarray) -> np.ndarray:
    pixels = np.ascontiguousarray(pixels, np.float32)
    r, c = pixels.shape
    out = np.zeros(r * c, np.float32)
    rc = lib().jxo_scaled_dct(r, c, pixels.ctypes.data, c, out.ctypes.data)
    assert rc == 0
    return out


def adjust_quant_bias(c: int, q: int, biases, rcp_mode: int = 0) -> float:
    b = np.ascontiguousarray(biases, np.float32)
    return float(lib().jxo_adjust_quant_bias(c, q, b.ctypes.data, rcp_mode))


def compute_sigma(desc: abi.FrameDesc) -> np.ndarray:
    s = desc.to_struct()
    out = np.zeros((desc.ysize_blocks + 4, desc.xsize_blocks + 4), np.float32)
    lib().jxo_compute_sigma(C.byref(s), out.ctypes.data)
    return out


def render_frame(desc: abi.FrameDesc, coeffs: np.ndarray, rcp_mode: int = 0) -> np.ndarray:
    """coeffs: (3, num_groups, 65536) int16|int32. Returns (H,W,3) or (3,H,W) per out_format."""
    want = np.int16 if desc.ac_type == abi.AC_INT16 else np.int32
    co = np.ascontiguousarray(coeffs, want)
    assert co.shape == (3, desc.num_groups, abi.GROUP_COEFFS), co.shape
    s = desc.to_struct()
    ptrs = (C.c_void_p * 3)(*[co.ctypes.data + c * co[0].nbytes for c in range(3)])
    out = np.zeros(desc.out_shape(desc.ysize), desc.out_dtype)   # (upsampled frames: out_ysize rows)
    rc = lib().jxo_render_frame(C.byref(s), ptrs, rcp_mode, out.ctypes.data)
    if rc:
        raise RuntimeError(f"jxo_render_frame rc={rc}")
    return out


def noise_planes(visible: int, nonvisible: int, w: int, h: int) -> np.ndarray:
    """Random3Planes before the convolution: (3, h, w) float32 in [1, 2), one generator per 256x256 output tile."""
    out = np.zeros((3, h, w), np.float32)
    lib().jxo_noise_planes(visible, nonvisible, w, h, out.ctypes.data)
    return out


def srgb_from_linear(v: np.ndarray) -> np.ndarray:
    """TF_SRGB::EncodedFromDisplay, element-wise (small arrays: scalar calls)."""
    fn = lib().jxo_srgb_from_linear
    flat = np.ascontiguousarray(v, np.float32).ravel()
    return np.array([fn(float(x)) for x in flat], np.float32).reshape(np.shape(v))


def make_unsigned(v: float, bits: int, x: int, y: int, c: int) -> int:
    return int(lib().jxo_make_unsigned(float(v), bits, x, y, c))


def f16_from_f32(v: np.ndarray) -> np.ndarray:
    fn = lib().jxo_f16_from_f32
    flat = np.ascontiguousarray(v, np.float32).ravel()
    return np.array([fn(float(x)) for x in flat], np.uint16).reshape(np.shape(v))


def dequant_dc(q: np.ndarray, dc_factors, mul: float, cfl_factors) -> np.ndarray:
    """q: (3, ys, xs) int32 quantised DC (X, Y, B). Returns (3, ys, xs) float32."""
    q = np.ascontiguousarray(q, np.int32)
    _, ys, xs = q.shape
    out = np.zeros(q.shape, np.float32)
    ptrs = (C.c_void_p * 3)(*[q.ctypes.data + c * q[0].nbytes for c in range(3)])
    f = (C.c_float * 3)(*dc_factors)
    cf = (C.c_float * 3)(*cfl_factors)
    lib().jxo_dequant_dc(ptrs, xs, ys, f, mul, cf, out.ctypes.data)
    return out


def adaptive_dc_smoothing(dc: np.ndarray, dc_factors) -> np.ndarray:
    dc = np.array(dc, np.float32, order="C")
    _, ys, xs = dc.shape
    f = (C.c_float * 3)(*dc_factors)
    rc = lib().jxo_adaptive_dc_smoothing(f, dc.ctypes.data, xs, ys)
    if rc:
        raise RuntimeError(f"jxo_adaptive_dc_smoothing rc={rc}")
    return dc


def desc_from_dump(d, **overrides) -> abi.FrameDesc:
    """FrameDesc from an oracle.ref.FrameDump (the reference decoder's own state)."""
    i = d.info
    acs = d.ac_strategy
    quant = np.where(acs & 1, d.raw_quant, 0).astype(np.int32)  # only first blocks are defined
    desc = abi.FrameDesc(
        xsize=i.xsize, ysize=i.ysize, ac_strategy=acs, raw_quant=quant, dc=d.dc,
        ytox=d.ytox, ytob=d.ytob, dequant=d.dequant, dequant_offsets=d.dequant_offsets,
        inv_global_scale=i.inv_global_scale, quant_scale=i.global_scale_float,
        x_dm_multiplier=i.x_dm_multiplier, b_dm_multiplier=i.b_dm_multiplier,
        quant_biases=tuple(i.quant_biases),
        cfl_base_x=i.cfl_base_x, cfl_base_b=i.cfl_base_b, cfl_color_scale=i.cfl_color_scale,
        gab=i.gab, gab_weights=tuple(i.gab_weights), epf_iters=i.epf_iters,
        epf_sharpness=d.sharpness, epf_sharp_lut=tuple(i.epf_sharp_lut),
        epf_channel_scale=tuple(i.epf_channel_scale), epf_quant_mul=i.epf_quant_mul,
        epf_pass0_sigma_scale=i.epf_pass0_sigma_scale, epf_pass2_sigma_scale=i.epf_pass2_sigma_scale,
        epf_border_sad_mul=i.epf_border_sad_mul,
        inverse_opsin_matrix=tuple(i.inverse_opsin_matrix),
        opsin_biases=tuple(i.opsin_biases)[:3], opsin_biases_cbrt=tuple(i.opsin_biases_cbrt)[:3],
        ac_type=abi.AC_INT16 if i.ac_is16 else abi.AC_INT32,
    )
    if getattr(i, "ycbcr", 0):
        desc.color_transform = 1
    if getattr(i, "noise", 0):
        desc.noise, desc.noise_lut = 1, tuple(i.noise_lut)
        desc.visible_frame_index, desc.nonvisible_frame_index = int(i.visible_frame_index), int(i.nonvisible_frame_index)
    if getattr(i, "upsampling", 1) > 1:
        desc.upsampling = int(i.upsampling)
        desc.upsampling_weights = np.array(list(i.upsampling_weights), np.float32)
        desc.xsize_upsampled, desc.ysize_upsampled = int(i.xsize_upsampled), int(i.ysize_upsampled)
    for k, v in overrides.items():
        setattr(desc, k, v)
    return desc
