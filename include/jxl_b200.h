/* jxl_b200.h -- C ABI of the GPU-native (H100) JPEG XL VarDCT decode transform pipeline.
 *
 * Drop-in boundary (SURVEY.md §8b).  libjxl keeps parsing headers and running the
 * ANS entropy decoder on the host under its own JxlParallelRunner
 * (lib/include/jxl/parallel_runner.h:127-129); instead of dequantising and
 * inverse-transforming each varblock on the CPU it hands the *quantised
 * coefficient groups + side information* to this library, which runs
 *
 *   dequant + chroma-from-luma + LLF-from-DC + variable-size IDCT   (replaces lib/jxl/dec_group.cc:431-450,
 *                                                                    dec_transforms-inl.h, dct-inl.h)
 *   Gaborish                                                        (replaces render_pipeline/stage_gaborish.cc:56-100)
 *   EPF pass 0 / 1 / 2 (+ sigma)                                    (replaces render_pipeline/stage_epf.cc, epf.cc:39-133)
 *   XYB -> linear RGB                                               (replaces render_pipeline/stage_xyb.cc:78-98,
 *                                                                    dec_xyb-inl.h:38-86)
 *   optional: linear -> sRGB transfer function                      (replaces render_pipeline/stage_from_linear.cc:42-53,
 *                                                                    cms/transfer_functions-inl.h:244-267)
 *   output packing f32 / f16 / u16 / dithered u8, RGB or RGBA       (replaces render_pipeline/stage_write.cc:455-640)
 *
 * as hand-written sm_90a CUDA kernels and returns the finished frame.
 *
 * Conventions: plain C, caller-owned pointers, no exceptions, every entry point
 * returns 0 on success or a JXLGPU_ERR_* code (the same "0 / non-zero" contract
 * as JxlParallelRetCode, parallel_runner.h:52-63) so that the host can fall back
 * to its CPU path (jxl::Status false) on any failure.  One frame in flight per
 * context.  Thread-safety: jxlgpu_submit_group may be called concurrently from
 * the runner's worker threads with distinct `thread_id` (< num_host_threads);
 * everything else is single-threaded per context, matching who calls what in
 * FrameDecoder (dec_frame.cc:573-735: frame_begin after ProcessACGlobal,
 * submit_group from ProcessACGroup, frame_finish from FinalizeFrame).
 */
#ifndef JXL_B200_H_
#define JXL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define JXLGPU_API __attribute__((visibility("default")))
#else
#define JXLGPU_API
#endif

#define JXLGPU_ABI_VERSION 6

enum {
  JXLGPU_OK = 0,
  JXLGPU_ERR_INVALID_ARGUMENT = 1,
  JXLGPU_ERR_UNSUPPORTED = 2,   /* frame not eligible: host must use its CPU path */
  JXLGPU_ERR_NO_DEVICE = 3,     /* CUDA device / driver missing: never a silent CPU fallback */
  JXLGPU_ERR_CUDA = 4,
  JXLGPU_ERR_OUT_OF_MEMORY = 5,
  JXLGPU_ERR_STATE = 6          /* call out of order (e.g. submit before frame_begin) */
};

/* Coefficient storage type, = jxl::ACType (lib/jxl/dct_util.h:41): libjxl picks
 * int16 when max_num_bits_ac < 16 (dec_frame.cc:417-431), int32 otherwise and
 * always int32 on the encoder-roundtrip caller (dec_group.cc:668). */
enum { JXLGPU_AC_INT16 = 0, JXLGPU_AC_INT32 = 1 };

/* Output pixel layouts. */
enum {
  JXLGPU_OUT_RGB_F32 = 0,       /* interleaved linear RGB float32, what JxlDecoderSetImageOutBuffer
                                   delivers for {3, JXL_TYPE_FLOAT} (decode.h:1021, types.h:80-104) */
  JXLGPU_OUT_PLANAR_F32 = 1,    /* 3 planes [c][y][x]; also used for intermediate-stage taps */
  /* The packed formats of WriteToOutputStage (stage_write.cc:455-640), native endianness, no
   * orientation change.  Unsigned: v*(2^bits-1), clamp, round-half-even (MakeUnsigned, :455-479);
   * 8-bit adds the reference's 32x32 ordered dither (:466-471).  Row stride >= xsize * pixel bytes. */
  JXLGPU_OUT_RGB_U8 = 2,        /* {3, JXL_TYPE_UINT8}: what djxl writes for 8-bit images */
  JXLGPU_OUT_RGBA_U8 = 3,       /* {4, JXL_TYPE_UINT8}, opaque alpha (no alpha channel on this path) */
  JXLGPU_OUT_RGB_U16 = 4,       /* {3, JXL_TYPE_UINT16} */
  JXLGPU_OUT_RGB_F16 = 5        /* {3, JXL_TYPE_FLOAT16}: round-to-nearest-even demotion (:590-640) */
};

/* Stage selection bits for jxlgpu_frame.stage_mask (0 = derive from gab/epf_iters,
 * i.e. the order PassesDecoderState::PreparePipeline builds, dec_cache.cc:151-170). */
enum {
  JXLGPU_STAGE_GAB = 1,
  JXLGPU_STAGE_EPF0 = 2,
  JXLGPU_STAGE_EPF1 = 4,
  JXLGPU_STAGE_EPF2 = 8,
  JXLGPU_STAGE_XYB = 16,
  JXLGPU_STAGE_SRGB = 32,  /* FromLinearStage<OpRgb>: sRGB OETF after XYB (stage_from_linear.cc:42-53).
                              Not part of the derived chain: OR it into stage_mask (alone, = derived
                              chain + transfer function, or together with EXPLICIT) when the output
                              colour encoding's transfer function is sRGB (stage_from_linear.cc:161-166) */
  JXLGPU_STAGE_EXPLICIT = 1u << 31 /* set to make stage_mask authoritative (test taps) */
};

#define JXLGPU_NUM_STRATEGIES 27   /* AcStrategy::kNumValidStrategies, ac_strategy.h:93-94 */
#define JXLGPU_GROUP_DIM 256       /* kGroupDim, frame_dimensions.h:25 */
#define JXLGPU_GROUP_COEFFS 65536  /* coefficients per group and channel */

typedef struct jxlgpu_ctx jxlgpu_ctx;

typedef struct jxlgpu_config {
  uint32_t abi_version;       /* JXLGPU_ABI_VERSION */
  int32_t device;             /* CUDA device ordinal */
  uint32_t num_host_threads;  /* upper bound of thread_id in submit_group (one upload stream each) */
  uint32_t flags;             /* reserved, 0 */
} jxlgpu_config;

/* Everything the hot path reads, as it sits in PassesSharedState / PassesDecoderState
 * after ProcessACGlobal (passes_state.h:48-96, dec_cache.h:86-188).  All plane
 * pointers are HOST pointers here; strides in elements.  Pageable planes are copied before
 * frame_begin returns; page-locked ones (jxlgpu_alloc_pinned) are read asynchronously and must stay
 * unchanged until frame_finish. */
typedef struct jxlgpu_frame {
  /* geometry: FrameDimensions (frame_dimensions.h:34-60) */
  uint32_t xsize, ysize;                /* true image size = mirror boundary of the filters */
  uint32_t xsize_blocks, ysize_blocks;  /* ceil(size/8) */
  uint32_t ac_type;                     /* JXLGPU_AC_* */
  /* row band rendered by this context, in AC-group rows (multi-GPU sharding, §8e).
   * band_ny_groups == 0 means the whole frame. Output rows are relative to the band. */
  uint32_t band_y0_groups, band_ny_groups;

  /* per 8x8-block planes [ysize_blocks][xsize_blocks] */
  const uint8_t* ac_strategy;   size_t ac_strategy_stride;  /* (type<<1)|is_first, ac_strategy.h:187-198 */
  const int32_t* raw_quant;     size_t raw_quant_stride;    /* valid at first blocks; [1,256] */
  const uint8_t* epf_sharpness; size_t epf_sharpness_stride;/* 0..7; may be NULL when epf_iters==0 */
  /* per 64x64-px tile chroma-from-luma factors (chroma_from_luma.h:135-136) */
  const int8_t* ytox_map; const int8_t* ytob_map; size_t cmap_stride;
  /* dequantised, smoothed DC, 3 planes [ysize_blocks][xsize_blocks] (compressed_dc.cc:128-300) */
  const float* dc[3];           size_t dc_stride;

  /* DequantMatrices table (quant_weights.h:364-367): matrix of strategy k, channel c starts
   * at dequant_table[dequant_offsets[3*k+c]] (a multiple of 4) and has 64*covered_blocks entries. */
  const float* dequant_table;   size_t dequant_table_floats;
  uint32_t dequant_offsets[3 * JXLGPU_NUM_STRATEGIES];

  /* scalars of DequantBlock (dec_group.cc:155-181) */
  float inv_global_scale;       /* Quantizer::InvGlobalScale() */
  float quant_scale;            /* Quantizer::Scale() (sigma, epf.cc:44,69) */
  float x_dm_multiplier, b_dm_multiplier;  /* dec_cache.h:161-162 */
  float quant_biases[4];        /* OpsinParams::quant_biases */
  float cfl_base_x, cfl_base_b; /* ColorCorrelation base_correlation_{x,b} */
  float cfl_color_scale;        /* 1 / color_factor (chroma_from_luma.h:51-57) */

  /* LoopFilter (loop_filter.h:20-70) */
  uint32_t gab;
  float gab_weights[6];         /* x1 x2 y1 y2 b1 b2 (unnormalised, as in the bitstream) */
  uint32_t epf_iters;
  float epf_sharp_lut[8];
  float epf_channel_scale[3];
  float epf_quant_mul, epf_pass0_sigma_scale, epf_pass2_sigma_scale, epf_border_sad_mul;

  /* OpsinParams (dec_xyb.h:28-34); matrix row-major, already x 255/intensity_target */
  float inverse_opsin_matrix[9];
  float opsin_biases[3];
  float opsin_biases_cbrt[3];

  uint32_t out_format;          /* JXLGPU_OUT_* */
  uint32_t stage_mask;          /* 0, JXLGPU_STAGE_SRGB, or JXLGPU_STAGE_EXPLICIT | bits */

  /* Optional DC stage on the device (the step in front of the path).  When quant_dc[0] != NULL the
   * `dc` planes above are not read: the library runs DequantDC (4:4:4 branch, compressed_dc.cc:199-232)
   * and, if dc_smoothing, AdaptiveDCSmoothing (compressed_dc.cc:50-197; FinalizeDC, dec_frame.cc:342-360)
   * itself.  quant_dc[c]: quantised DC of channel X, Y, B per 8x8 block = modular channels 1, 0, 2 of
   * the VarDCT DC groups (dec_modular.cc:446-449), frame-wide planes. */
  const int32_t* quant_dc[3];
  size_t quant_dc_stride;       /* elements */
  float dc_factors[3];          /* quantizer.MulDC() (quantizer.h:140) */
  float dc_cfl_factors[3];      /* cmap.base().DCFactors() (dec_modular.cc:462) */
  const float* dc_group_mul;    /* per DC group (2048x2048 px, raster order) 1 / (1 << extra_precision)
                                   (dec_modular.cc:443-444); NULL = 1 everywhere */
  uint32_t dc_smoothing;        /* 0 when kSkipAdaptiveDCSmoothing or kUseDcFrame is set */

  /* Upsampling (SURVEY.md §8f rank 4; UpsamplingStage, lib/jxl/render_pipeline/stage_upsampling.cc:51-271,
   * placed after the filters and before XYB->RGB by PreparePipeline, dec_cache.cc:216-227).
   * upsampling: frame_header.upsampling = 1 (or 0: none), 2, 4 or 8.  Everything above (xsize, blocks,
   * filters) is at the coded resolution; the output buffer is xsize_upsampled x ysize_upsampled
   * (FrameDimensions::{x,y}size_upsampled, <= upsampling * size; 0 = upsampling * size).
   * upsampling_weights: CustomTransformData::upsampling{2,4,8}_weights of that factor (15 / 55 / 210 floats,
   * image_metadata.h:193-196), read by frame_begin.  Whole-frame contexts only (band_ny_groups == 0). */
  uint32_t upsampling;
  uint32_t xsize_upsampled, ysize_upsampled;
  const float* upsampling_weights;

  /* Noise (SURVEY.md §8f rank 4): frame_header.flags & kNoise.  The library generates the three noise planes on
   * the device (Random3Planes, lib/jxl/dec_noise.cc:45-152: Xorshift128Plus per 256x256 tile of the output image,
   * seeded with the two frame indices of PassesDecoderState (dec_cache.h:127-128) and the tile origin), convolves
   * them (ConvolveNoiseStage, stage_noise.cc:263-304) and mixes them into X, Y, B with the strength LUT
   * (AddNoiseStage, :140-251; NoiseParams::lut, noise.h:27-43; the chroma factors are cfl_base_x / cfl_base_b)
   * after the filters and the upsampling, before XYB -> RGB (dec_cache.cc:232-236).  Whole-frame contexts only. */
  uint32_t noise;
  float noise_lut[8];
  uint32_t visible_frame_index, nonvisible_frame_index;

  /* Colour transform of the frame (frame_header.color_transform): 0 = XYB (everything above), 1 = YCbCr --
   * JPEG-origin frames without chroma subsampling (4:4:4): the colour stage (JXLGPU_STAGE_XYB position) is then
   * kYCbCrStage (lib/jxl/render_pipeline/stage_ycbcr.cc:33-71, full-range BT.601; channel 0 = Cb, 1 = Y, 2 = Cr) and
   * its output is already in the image's own (non-linear) encoding: no JXLGPU_STAGE_SRGB. */
  uint32_t color_transform;
  uint32_t reserved1;
} jxlgpu_frame;

JXLGPU_API uint32_t jxlgpu_abi_version(void);
JXLGPU_API const char* jxlgpu_error_string(int code);
/* Last CUDA error text recorded by this context (for logs). */
JXLGPU_API const char* jxlgpu_last_error(const jxlgpu_ctx* ctx);

JXLGPU_API int jxlgpu_create(jxlgpu_ctx** ctx, const jxlgpu_config* config);
JXLGPU_API void jxlgpu_destroy(jxlgpu_ctx* ctx);

/* Starts a frame: validates eligibility, (re)sizes device buffers, uploads side info.
 * Replaces the per-frame setup in DecodeGroupImpl (dec_group.cc:183-228). */
JXLGPU_API int jxlgpu_frame_begin(jxlgpu_ctx* ctx, const jxlgpu_frame* frame);

/* Optional, right after frame_begin: announce the host output buffer (what libjxl knows since
 * JxlDecoderSetImageOutBuffer, decode.h:1021).  Finished AC-group rows are then copied back
 * while later groups are still being submitted; frame_finish(out) with the same pointer only
 * waits.  Layout as in frame_finish. */
JXLGPU_API int jxlgpu_frame_set_output(jxlgpu_ctx* ctx, void* out, size_t out_stride_bytes);

/* One entropy-decoded AC group: coeff[c] points at `ncoeff` quantised coefficients of
 * channel c (X, Y, B) in libjxl's ACImage order -- varblocks in raster order of their
 * first block, each 64*covered_blocks long (dec_group.cc:335-359).  Asynchronous H2D on
 * the stream of `thread_id`: pinned buffers must stay valid until frame_finish, pageable ones
 * are staged by the driver before the call returns.  If the three channel buffers are one
 * contiguous [3][65536] block (coeff[c] == coeff[0] + c*65536 elements -- e.g. an ACImage subclass
 * over pinned memory, lib/jxl/dct_util.h:43-91) the group travels as a single DMA.  When the last group of an AC-group row
 * arrives, that row's kernels are enqueued right away (see jxl_b200.cu).
 * Replaces dec_group.cc:431-450 + RenderPipelineInput::Done(). */
JXLGPU_API int jxlgpu_submit_group(jxlgpu_ctx* ctx, uint32_t group_idx, size_t thread_id,
                                   const void* const coeff[3], size_t ncoeff);

/* Same, for `n` groups in one call: coeff[3*i + c] is channel c of group group_idx[i]. */
JXLGPU_API int jxlgpu_submit_groups(jxlgpu_ctx* ctx, size_t n, const uint32_t* group_idx, size_t thread_id,
                                    const void* const* coeff, const size_t* ncoeff);

/* Sparse hand-off: only the NON-ZERO quantised coefficients of an AC group cross PCIe (at d >= 1
 * about 85-90% of them are zero, so this is 5-8x fewer bytes than the dense planes).  It is what
 * the entropy decoder's inner loop produces anyway: DecodeACVarBlock visits the non-zeros one by
 * one (`block[order[k]] += coeff`, dec_group.cc:515-534) into a block it had to zero-fill first
 * (:341-355); with this entry point it appends `(offset + order[k]) << 16 | (uint16_t)coeff` to a
 * per-group list instead and skips the zero-fill.
 *   nz16[c]: n16[c] words `(pos << 16) | (uint16_t)value`, -32768 <= value <= 32767
 *   nz32[c]: n32[c] pairs of words `{pos, (uint32_t)value}` for larger values (int32 frames only)
 * pos = index of the coefficient inside the group's channel plane (< 65536; same order as the dense
 * layout of jxlgpu_submit_group), entries in any order, every pos at most once (single pass).  The
 * library zero-fills the group's dense planes in HBM, copies the lists (adjacent host arrays travel
 * as one DMA) and expands them with a scatter kernel on the upload stream. */
typedef struct jxlgpu_sparse_group {
  uint32_t group_idx;
  uint32_t n16[3];
  uint32_t n32[3];
  const uint32_t* nz16[3];
  const uint32_t* nz32[3];
} jxlgpu_sparse_group;

JXLGPU_API int jxlgpu_submit_groups_sparse(jxlgpu_ctx* ctx, size_t n, const jxlgpu_sparse_group* groups,
                                           size_t thread_id);

/* Runs the kernels for every submitted group of the band and copies the band's pixels to
 * `out` (host; row stride in bytes).  out == NULL keeps the result on the device
 * (jxlgpu_device_output).  Replaces LowMemoryRenderPipeline::ProcessBuffers + the write
 * stage for the in-scope stages (low_memory_render_pipeline.cc:832-934). */
JXLGPU_API int jxlgpu_frame_finish(jxlgpu_ctx* ctx, void* out, size_t out_stride_bytes);

/* ---- device-resident entry points (bench / multi-GPU plumbing; pointers are DEVICE) ---- */

/* Use coefficient planes that already live in HBM: dev_coeff[c] = [num_groups][65536]
 * elements of the frame's ac_type.  Marks every group as submitted.  Each plane must be aligned to
 * the element size (2 bytes for int16, 4 for int32): jxlgpu_render_device / jxlgpu_frame_finish
 * return JXLGPU_ERR_INVALID_ARGUMENT otherwise, before enqueuing anything.  16-byte aligned planes
 * select the bulk-copy 8x8 kernel; others are read with ordinary loads, which is slower. */
JXLGPU_API int jxlgpu_set_device_coefficients(jxlgpu_ctx* ctx, const void* const dev_coeff[3]);
/* Enqueue the whole hot path on `cuda_stream` (a cudaStream_t, 0 = context stream) writing
 * the band to dev_out (device pointer or NULL for the context's own buffer). No host sync. */
JXLGPU_API int jxlgpu_render_device(jxlgpu_ctx* ctx, void* dev_out, size_t out_stride_bytes,
                                    void* cuda_stream);
/* Multi-GPU fused all-gather.  dev_ptrs[i] (i < n <= 8) are addresses -- valid on THIS device, i.e.
 * peer-mapped over NVLink -- of this band's slot inside the other ranks' frame buffers; `dev_out` of
 * jxlgpu_render_device is the same slot in the local frame buffer.  Every filter CTA, after writing its
 * strip segment locally, replays it to all of them with wide coalesced stores, so the gather overlaps
 * the filtering and no collective kernel runs.  If multicast_ptr is non-NULL it is the slot's NVSwitch
 * multicast address and one multimem.st.v2 per 8 bytes replaces the n stores.  n = 0 and NULL switch it
 * off.  The caller owns the cross-GPU barrier that publishes the frame (bench.py: symmetric-memory
 * barrier).  Only the production stage chains (filter_strip_kernel) replicate. */
JXLGPU_API int jxlgpu_set_output_replicas(jxlgpu_ctx* ctx, uint32_t n, void* const* dev_ptrs, void* multicast_ptr);
/* Context-owned output buffer of the last render (device pointer) and its row stride. */
JXLGPU_API int jxlgpu_device_output(jxlgpu_ctx* ctx, void** dev_ptr, size_t* stride_bytes);
/* Post-IDCT XYB planes [3][ysize_blocks*8][xsize_blocks*8], row-major (device pointer): halo
 * exchange between bands and stage taps.  The renders keep this intermediate in 8x8 block tiles; the
 * call synchronises with the last render, copies it into a context-owned row-major buffer (one
 * kernel launch) and returns that buffer, valid until the next call, frame_begin or destroy. */
JXLGPU_API int jxlgpu_device_xyb(jxlgpu_ctx* ctx, float** dev_ptr, size_t* plane_stride_floats,
                                 size_t* row_stride_floats);
JXLGPU_API int jxlgpu_synchronize(jxlgpu_ctx* ctx);
/* Number of kernel launches issued by this context since creation (bench "gpu_launches"). */
JXLGPU_API uint64_t jxlgpu_launch_count(const jxlgpu_ctx* ctx);
/* Per-kernel device times of the LAST render (ms): plan, 8x8-class IDCT, mid IDCT (16/32),
 * large IDCT (64+), filter.
 * Measured with CUDA events recorded on the launch stream; enable before rendering. */
JXLGPU_API int jxlgpu_set_profiling(jxlgpu_ctx* ctx, int enable);
JXLGPU_API int jxlgpu_kernel_times(jxlgpu_ctx* ctx, float ms[5]);
/* Page-locked host memory for coefficient / output staging (truly asynchronous copies). */
JXLGPU_API void* jxlgpu_alloc_pinned(size_t bytes);
JXLGPU_API void jxlgpu_free_pinned(void* p);

#ifdef __cplusplus
}
#endif
#endif /* JXL_B200_H_ */
