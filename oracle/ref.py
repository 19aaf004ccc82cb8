"""ctypes binding of oracle/_ref/libjxl_ref_harness.so (the UNMODIFIED reference,
built by oracle/build_ref.py).  TEST INFRASTRUCTURE ONLY: importable from tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
Never imported by the product package `libjxl_b200`.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
SO = HERE / "_ref" / "libjxl_ref_harness.so"
# Same sources built with -ffp-contract=off (FMA only where the source says MulAdd):
# the bit-exact pin for oracle/jxl_oracle.c.  Select with use_variant("strict").
SO_STRICT = HERE / "_ref" / "libjxl_ref_harness_strict.so"
# The reference with the jxl_b200 backend compiled in (build-time patched copies of dec_frame.cc /
# dec_group.cc + integration/libjxl_gpu_backend.h, linked against libjxl_b200.so): use_variant("gpu").
SO_GPU = HERE / "_ref" / "libjxl_ref_harness_gpu.so"
_SO = {"default": SO, "strict": SO_STRICT, "gpu": SO_GPU}


class RefFrameInfo(C.Structure):
    _fields_ = [
        ("xsize", C.c_int32), ("ysize", C.c_int32),
        ("xsize_blocks", C.c_int32), ("ysize_blocks", C.c_int32),
        ("xsize_groups", C.c_int32), ("ysize_groups", C.c_int32),
        ("num_groups", C.c_int32), ("ac_is16", C.c_int32),
        ("cmap_xsize", C.c_int32), ("cmap_ysize", C.c_int32),
        ("gab", C.c_int32), ("epf_iters", C.c_int32),
        ("inv_global_scale", C.c_float), ("global_scale_float", C.c_float),
        ("x_dm_multiplier", C.c_float), ("b_dm_multiplier", C.c_float),
        ("quant_biases", C.c_float * 4),
        ("cfl_base_x", C.c_float), ("cfl_base_b", C.c_float), ("cfl_color_scale", C.c_float),
        ("gab_weights", C.c_float * 6),
        ("epf_sharp_lut", C.c_float * 8),
        ("epf_channel_scale", C.c_float * 3),
        ("epf_quant_mul", C.c_float), ("epf_pass0_sigma_scale", C.c_float),
        ("epf_pass2_sigma_scale", C.c_float), ("epf_border_sad_mul", C.c_float),
        ("inverse_opsin_matrix", C.c_float * 9),
        ("opsin_biases", C.c_float * 4),
        ("opsin_biases_cbrt", C.c_float * 4),
        ("dequant_table_floats", C.c_int32),
        ("dequant_offsets", C.c_int32 * 81),
        ("upsampling", C.c_int32), ("xsize_upsampled", C.c_int32), ("ysize_upsampled", C.c_int32),
        ("upsampling_weights", C.c_float * 210),
        ("ycbcr", C.c_int32),
        ("noise", C.c_int32), ("noise_lut", C.c_float * 8),
        ("visible_frame_index", C.c_uint32), ("nonvisible_frame_index", C.c_uint32),
    ]


class RefFrameParams(C.Structure):
    """ref_frame_set_params: frame-header / image-metadata values written into an opened frame."""
    _fields_ = [
        ("x_dm_multiplier", C.c_float), ("b_dm_multiplier", C.c_float),
        ("quant_biases", C.c_float * 4),
        ("cfl_base_x", C.c_float), ("cfl_base_b", C.c_float), ("color_factor", C.c_uint32),
        ("gab_weights", C.c_float * 6),
        ("epf_sharp_lut", C.c_float * 8),
        ("epf_channel_scale", C.c_float * 3),
        ("epf_quant_mul", C.c_float), ("epf_pass0_sigma_scale", C.c_float),
        ("epf_pass2_sigma_scale", C.c_float), ("epf_border_sad_mul", C.c_float),
        ("inverse_opsin_matrix", C.c_float * 9),
        ("opsin_biases", C.c_float * 3),
    ]


PLANE_AC_STRATEGY, PLANE_RAW_QUANT, PLANE_SHARPNESS, PLANE_YTOX, PLANE_YTOB = 0, 1, 2, 3, 4
PLANE_DC, PLANE_SIGMA, PLANE_DEQUANT, PLANE_COEFFS, PLANE_DECODED = 5, 6, 7, 8, 9

STAGE_GAB, STAGE_EPF0, STAGE_EPF1, STAGE_EPF2, STAGE_XYB = 1, 2, 4, 8, 16
STAGE_UPSAMPLING = 64   # ref_frame_render: the frame's own UpsamplingStage (before XYB)
STAGE_NOISE = 128        # ref_frame_render: ConvolveNoise + AddNoise of a frame with the kNoise flag

_libs: dict = {}
_variant = "default"


def available(variant: str = "default") -> bool:
    return _SO[variant].exists()


def can_set_params() -> bool:
    """Whether the selected harness build has ref_frame_set_params (Frame.set_params).  A prebuilt oracle/_ref
    made from an older harness, on a machine without the reference sources to rebuild it, does not."""
    return hasattr(lib(), "ref_frame_set_params")


def can_set_ups_noise() -> bool:
    """Whether the selected harness build has ref_frame_set_upsampling_weights and ref_frame_set_noise_lut
    (Frame.set_upsampling_weights / set_noise_lut); an older prebuilt oracle/_ref does not."""
    return hasattr(lib(), "ref_frame_set_upsampling_weights") and hasattr(lib(), "ref_frame_set_noise_lut")


def use_variant(variant: str) -> None:
    """'default' = the reference's own build flags; 'strict' = + -ffp-contract=off."""
    global _variant
    assert variant in _SO
    _variant = variant


def lib():
    if _variant not in _libs:
        so = _SO[_variant]
        if not so.exists():
            raise RuntimeError(f"{so} missing: run `python oracle/build_ref.py` where /root/reference exists")
        L = C.CDLL(str(so))
        L.ref_frame_open.restype = C.c_void_p
        L.ref_frame_open.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
        L.ref_frame_open_storage.restype = C.c_void_p
        L.ref_frame_open_storage.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int]
        from libjxl_b200 import abi as _abi
        L.ref_frame_bind_gpu_frame.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(_abi.JxlGpuFrame)]
        L.ref_frame_raw_coeffs.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        L.ref_frame_close.argtypes = [C.c_void_p]
        L.ref_frame_info.argtypes = [C.c_void_p, C.POINTER(RefFrameInfo)]
        if hasattr(L, "ref_frame_set_params"):   # (absent from a harness built before it existed)
            L.ref_frame_set_params.argtypes = [C.c_void_p, C.POINTER(RefFrameParams)]
        if hasattr(L, "ref_frame_set_upsampling_weights"):
            L.ref_frame_set_upsampling_weights.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        if hasattr(L, "ref_frame_set_noise_lut"):
            L.ref_frame_set_noise_lut.argtypes = [C.c_void_p, C.c_void_p]
        L.ref_frame_get_plane.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
        L.ref_frame_render.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_double)]
        L.ref_decode_native.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                        C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.ref_dequant_dc.argtypes = [C.c_void_p * 3, C.c_size_t, C.c_size_t, C.c_float * 3, C.c_float,
                                     C.c_float * 3, C.c_void_p]
        L.ref_adaptive_dc_smoothing.argtypes = [C.c_float * 3, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int]
        L.ref_frame_render_out.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                           C.POINTER(C.c_double)]
        L.ref_encode_rgb8_ex.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_int, C.POINTER(C.POINTER(C.c_uint8)),
                                         C.POINTER(C.c_size_t)]
        L.ref_decode_linear_f32.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p,
                                            C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.ref_runner_create.restype = C.c_void_p
        L.ref_runner_create.argtypes = [C.c_int]
        L.ref_runner_destroy.argtypes = [C.c_void_p]
        L.ref_free.argtypes = [C.c_void_p]
        if hasattr(L, "ref_gpu_frames_taken"):
            L.ref_gpu_frames_taken.restype = C.c_ulonglong
        if hasattr(L, "ref_hwy_target"):
            L.ref_hwy_target.restype = C.c_char_p
        L.ref_transform_to_pixels.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        L.ref_transform_from_pixels.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        L.ref_llf_from_dc.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        _libs[_variant] = L
    return _libs[_variant]


def encode_rgb8(img: np.ndarray, distance: float = 1.0, effort: int = 7, gaborish: int = -1,
                epf: int = -1, threads: int | None = None, resampling: int = -1) -> bytes:
    """cjxl-equivalent through the public JxlEncoder API; returns a bare codestream."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w, c = img.shape
    assert c == 3
    out = C.POINTER(C.c_uint8)()
    n = C.c_size_t()
    rc = lib().ref_encode_rgb8_ex(img.ctypes.data, w, h, distance, effort, gaborish, epf, resampling,
                                  threads or os.cpu_count() or 1, C.byref(out), C.byref(n))
    if rc:
        raise RuntimeError(f"ref_encode_rgb8 failed rc={rc}")
    data = C.string_at(out, n.value)
    lib().ref_free(out)
    return data


def encode_jpeg(jpeg: bytes, threads: int | None = None) -> bytes:
    """Lossless JPEG recompression through JxlEncoderAddJPEGFrame (YCbCr VarDCT frame); bare codestream."""
    out = C.POINTER(C.c_uint8)()
    n = C.c_size_t()
    L = lib()
    L.ref_encode_jpeg.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]
    rc = L.ref_encode_jpeg(jpeg, len(jpeg), threads or os.cpu_count() or 1, C.byref(out), C.byref(n))
    if rc:
        raise RuntimeError(f"ref_encode_jpeg failed rc={rc}")
    data = C.string_at(out, n.value)
    L.ref_free(out)
    return data


class Runner:
    def __init__(self, threads: int):
        self.threads = threads
        self.h = lib().ref_runner_create(threads)

    def close(self):
        if self.h:
            lib().ref_runner_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()


def decode_linear_f32(data: bytes, threads: int = 1, out: np.ndarray | None = None,
                      runner: Runner | None = None) -> np.ndarray:
    """Full reference decode (public API) -> (H, W, 3) linear sRGB float32."""
    w, h = C.c_int(), C.c_int()
    if out is None:
        rc = lib().ref_decode_linear_f32(data, len(data), runner.h if runner else None, threads,
                                         None, 0, C.byref(w), C.byref(h))
        if rc:
            raise RuntimeError(f"ref_decode_linear_f32 (probe) rc={rc}")
        out = np.empty((h.value, w.value, 3), np.float32)
    rc = lib().ref_decode_linear_f32(data, len(data), runner.h if runner else None, threads,
                                     out.ctypes.data, out.size, C.byref(w), C.byref(h))
    if rc:
        raise RuntimeError(f"ref_decode_linear_f32 rc={rc}")
    return out


@dataclass
class FrameDump:
    """Everything the hot path consumes, as the reference decoder produced it."""
    info: RefFrameInfo
    ac_strategy: np.ndarray   # u8  (yb, xb)
    raw_quant: np.ndarray     # i32 (yb, xb)
    sharpness: np.ndarray     # u8  (yb, xb)
    ytox: np.ndarray          # i8  (cmy, cmx)
    ytob: np.ndarray          # i8
    dc: np.ndarray            # f32 (3, yb, xb)
    sigma: np.ndarray | None  # f32 (yb+4, xb+4) inverse sigma, reference-computed
    dequant: np.ndarray       # f32 (table,)
    dequant_offsets: np.ndarray  # i32 (27, 3)
    coeffs: np.ndarray        # i16|i32 (3, num_groups, 65536)
    decoded: np.ndarray       # f32 (H, W, 3) reference decode, linear sRGB


class Frame:
    """A frame opened with the reference's FrameDecoder, coefficients retained."""

    def __init__(self, data: bytes, threads: int = 1, storage: int = 0):
        """storage 1: the reference's entropy decoder writes through integration/pinned_ac_image.h
        (group-major layout) instead of its own ACImageT."""
        self.h = None
        self.h = lib().ref_frame_open_storage(data, len(data), threads, storage)
        if not self.h:
            raise RuntimeError("ref_frame_open failed (frame not eligible for the hot path?)")
        self.info = RefFrameInfo()
        lib().ref_frame_info(self.h, C.byref(self.info))

    def bind_gpu_frame(self, out_format: int = 0, stage_mask: int = 0):
        """integration/gpu_frame_binding.h applied to the live decoder state: the jxlgpu_frame a libjxl
        host would pass to jxlgpu_frame_begin (pointers into the reference's images; valid until close)."""
        from libjxl_b200 import abi as _abi
        s = _abi.JxlGpuFrame()
        rc = lib().ref_frame_bind_gpu_frame(self.h, out_format, stage_mask, C.byref(s))
        if rc:
            raise RuntimeError(f"ref_frame_bind_gpu_frame rc={rc}")
        return s

    def set_params(self, hdr: dict) -> None:
        """Write a header set (jxl_workload.header_params: the HEADER_FIELDS plus color_factor) into the opened
        frame as if its bitstream had carried it; the sigma image is recomputed.  `info` (and so dump(),
        desc_from_dump and bind_gpu_frame) then reports the new values."""
        if not can_set_params():
            raise RuntimeError(f"{_SO[_variant]} predates ref_frame_set_params: rebuild it with `python oracle/build_ref.py`")
        p = RefFrameParams()
        for name, _ in RefFrameParams._fields_:
            v = hdr[name]
            if hasattr(getattr(p, name), "__len__"):
                getattr(p, name)[:] = [float(x) for x in v]
            else:
                setattr(p, name, v)
        rc = lib().ref_frame_set_params(self.h, C.byref(p))
        if rc:
            raise RuntimeError(f"ref_frame_set_params rc={rc}")
        lib().ref_frame_info(self.h, C.byref(self.info))

    def set_upsampling_weights(self, n: int, weights) -> None:
        """Custom upsampling weights of factor n (F16 values), read into the frame's CustomTransformData through
        the reference's Bundle reader."""
        if not can_set_ups_noise():
            raise RuntimeError(f"{_SO[_variant]} predates ref_frame_set_upsampling_weights: rebuild it with "
                               "`python oracle/build_ref.py`")
        w = np.ascontiguousarray(weights, np.float32)
        rc = lib().ref_frame_set_upsampling_weights(self.h, n, w.ctypes.data)
        if rc:
            raise RuntimeError(f"ref_frame_set_upsampling_weights rc={rc}")
        lib().ref_frame_info(self.h, C.byref(self.info))

    def set_noise_lut(self, lut) -> None:
        """The noise strength LUT (values k / 1024, k <= 1023), read through the reference's DecodeNoise; the frame
        must carry the noise flag."""
        if not can_set_ups_noise():
            raise RuntimeError(f"{_SO[_variant]} predates ref_frame_set_noise_lut: rebuild it with "
                               "`python oracle/build_ref.py`")
        v = np.ascontiguousarray(lut, np.float32)
        assert v.size == 8
        rc = lib().ref_frame_set_noise_lut(self.h, v.ctypes.data)
        if rc:
            raise RuntimeError(f"ref_frame_set_noise_lut rc={rc}")
        lib().ref_frame_info(self.h, C.byref(self.info))

    def raw_group_major_coeffs(self) -> np.ndarray:
        """storage 1 only: the allocation itself, viewed as (num_groups, 3, 65536) -- exactly the host
        blocks jxlgpu_submit_group(s) would be handed."""
        base, nbytes = C.c_void_p(), C.c_size_t()
        if lib().ref_frame_raw_coeffs(self.h, C.byref(base), C.byref(nbytes)):
            raise RuntimeError("frame was not opened with storage=1")
        dt = np.int16 if self.info.ac_is16 else np.int32
        buf = (C.c_uint8 * nbytes.value).from_address(base.value)
        return np.frombuffer(buf, dt).reshape(self.info.num_groups, 3, 65536)

    def close(self):
        if self.h:
            lib().ref_frame_close(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _plane(self, which: int, shape, dtype) -> np.ndarray:
        a = np.empty(shape, dtype)
        rc = lib().ref_frame_get_plane(self.h, which, a.ctypes.data, a.nbytes)
        if rc:
            raise RuntimeError(f"ref_frame_get_plane({which}) rc={rc}")
        return a

    def dump(self) -> FrameDump:
        i = self.info
        yb, xb = i.ysize_blocks, i.xsize_blocks
        sigma = None
        if i.epf_iters > 0:
            sigma = self._plane(PLANE_SIGMA, (yb + 4, xb + 4), np.float32)
        return FrameDump(
            info=i,
            ac_strategy=self._plane(PLANE_AC_STRATEGY, (yb, xb), np.uint8),
            raw_quant=self._plane(PLANE_RAW_QUANT, (yb, xb), np.int32),
            sharpness=self._plane(PLANE_SHARPNESS, (yb, xb), np.uint8),
            ytox=self._plane(PLANE_YTOX, (i.cmap_ysize, i.cmap_xsize), np.int8),
            ytob=self._plane(PLANE_YTOB, (i.cmap_ysize, i.cmap_xsize), np.int8),
            dc=self._plane(PLANE_DC, (3, yb, xb), np.float32),
            sigma=sigma,
            dequant=self._plane(PLANE_DEQUANT, (i.dequant_table_floats,), np.float32),
            dequant_offsets=np.array(list(i.dequant_offsets), np.int32).reshape(27, 3),
            coeffs=self._plane(PLANE_COEFFS, (3, i.num_groups, 65536),
                               np.int16 if i.ac_is16 else np.int32),
            decoded=self._plane(PLANE_DECODED, (i.ysize_upsampled, i.xsize_upsampled, 3), np.float32),
        )

    def render(self, stage_mask: int = -1, reps: int = 1, want_output: bool = True):
        """Hot path only (reference code) from the retained coefficients.
        Returns (planar f32 (3,H,W) or None, [seconds per rep])."""
        i = self.info
        ups = stage_mask >= 0 and (stage_mask & STAGE_UPSAMPLING) and i.upsampling > 1
        shape = (3, i.ysize_upsampled, i.xsize_upsampled) if ups else (3, i.ysize, i.xsize)
        out = np.empty(shape, np.float32) if want_output else None
        secs = (C.c_double * max(reps, 1))()
        rc = lib().ref_frame_render(self.h, stage_mask, out.ctypes.data if want_output else None,
                                    reps, secs)
        if rc:
            raise RuntimeError(f"ref_frame_render rc={rc}")
        return out, list(secs)


    _OUT = {0: ("float32", 3), 2: ("uint8", 3), 3: ("uint8", 4), 4: ("uint16", 3), 5: ("float16", 3)}

    def render_out(self, stage_mask: int = -1, out_format: int = 0, reps: int = 1, want_output: bool = True):
        """Hot path ending in the reference's FromLinear (stage_mask bit 32; -33 = derived chain +
        sRGB) and WriteToOutput stages.  out_format as JXLGPU_OUT_* (interleaved ones).
        Returns ((H, W, ch) array or None, [seconds per rep])."""
        i = self.info
        dt, ch = self._OUT[out_format]
        out = np.zeros((i.ysize, i.xsize, ch), dt) if want_output else None
        secs = (C.c_double * max(reps, 1))()
        rc = lib().ref_frame_render_out(self.h, stage_mask, out_format, out.ctypes.data if want_output else None,
                                        reps, secs)
        if rc:
            raise RuntimeError(f"ref_frame_render_out rc={rc}")
        return out, list(secs)


def transform_to_pixels(strategy: int, coeffs: np.ndarray, rows: int, cols: int) -> np.ndarray:
    coeffs = np.ascontiguousarray(coeffs, np.float32).ravel()
    px = np.zeros((rows, cols), np.float32)
    rc = lib().ref_transform_to_pixels(strategy, coeffs.ctypes.data, coeffs.size, px.ctypes.data, cols)
    if rc:
        raise RuntimeError(f"ref_transform_to_pixels rc={rc}")
    return px


def transform_from_pixels(strategy: int, pixels: np.ndarray) -> np.ndarray:
    pixels = np.ascontiguousarray(pixels, np.float32)
    rows, cols = pixels.shape
    co = np.zeros(rows * cols, np.float32)
    rc = lib().ref_transform_from_pixels(strategy, pixels.ctypes.data, cols, co.ctypes.data, co.size)
    if rc:
        raise RuntimeError(f"ref_transform_from_pixels rc={rc}")
    return co


def llf_from_dc(strategy: int, dc: np.ndarray, block: np.ndarray) -> np.ndarray:
    dc = np.ascontiguousarray(dc, np.float32)
    block = np.ascontiguousarray(block, np.float32).ravel().copy()
    rc = lib().ref_llf_from_dc(strategy, dc.ctypes.data, dc.shape[1], block.ctypes.data, block.size)
    if rc:
        raise RuntimeError(f"ref_llf_from_dc rc={rc}")
    return block


def dequant_dc(q: np.ndarray, dc_factors, mul: float, cfl_factors) -> np.ndarray:
    """jxl::DequantDC (4:4:4) on one DC group; q: (3, ys, xs) int32 in X, Y, B order."""
    q = np.ascontiguousarray(q, np.int32)
    _, ys, xs = q.shape
    out = np.zeros(q.shape, np.float32)
    ptrs = (C.c_void_p * 3)(*[q.ctypes.data + c * q[0].nbytes for c in range(3)])
    rc = lib().ref_dequant_dc(ptrs, xs, ys, (C.c_float * 3)(*dc_factors), mul, (C.c_float * 3)(*cfl_factors),
                              out.ctypes.data)
    if rc:
        raise RuntimeError(f"ref_dequant_dc rc={rc}")
    return out


def adaptive_dc_smoothing(dc: np.ndarray, dc_factors, threads: int = 1) -> np.ndarray:
    """jxl::AdaptiveDCSmoothing on a (3, ys, xs) DC image (returns a new array)."""
    dc = np.array(dc, np.float32, order="C")
    _, ys, xs = dc.shape
    rc = lib().ref_adaptive_dc_smoothing((C.c_float * 3)(*dc_factors), dc.ctypes.data, xs, ys, threads)
    if rc:
        raise RuntimeError(f"ref_adaptive_dc_smoothing rc={rc}")
    return dc


_NATIVE = {"float32": 0, "uint8": 2, "uint16": 3, "float16": 5}   # JxlDataType, jxl/types.h


def decode_native(data: bytes, shape, dtype, threads: int = 1) -> np.ndarray:
    """Public-API decode with no output colour profile override (what djxl does by default) into an
    (H, W, channels) array of `dtype`."""
    out = np.zeros(shape, dtype)
    w, h = C.c_int(0), C.c_int(0)
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    rc = lib().ref_decode_native(buf, len(data), threads, _NATIVE[np.dtype(dtype).name], shape[2], out.ctypes.data,
                                 out.nbytes, C.byref(w), C.byref(h))
    if rc:
        raise RuntimeError(f"ref_decode_native rc={rc}")
    assert (h.value, w.value) == tuple(shape[:2]), (h.value, w.value, shape)
    return out


def hwy_target() -> str:
    """Highway target the reference's dynamic dispatch runs on this CPU (e.g. 'AVX2')."""
    L = lib()
    return L.ref_hwy_target().decode() if hasattr(L, "ref_hwy_target") else "unknown"


def gpu_frames_taken() -> int:
    """'gpu' variant: frames the compiled-in jxl_b200 backend has rendered in this process."""
    L = lib()
    return int(L.ref_gpu_frames_taken()) if hasattr(L, "ref_gpu_frames_taken") else 0
