// jxl_kernels.cuh -- sm_90a (Hopper) kernels of the JPEG XL VarDCT decode transform pipeline.
//
// Written from scratch; the arithmetic contract (operation order,
// explicit FMAs) is the reference's, cited per function as /root/reference paths:
//   dequant + CfL            lib/jxl/dec_group.cc:115-181, lib/jxl/quantizer-inl.h:35-67
//   LLF from DC              lib/jxl/dec_transforms-inl.h:35-64,691-818
//   1-D (I)DCT recursion     lib/jxl/dct-inl.h:45-232   (Perera-Liu radix-2)
//   2-D transforms, specials lib/jxl/dct-inl.h:349-397, lib/jxl/dec_transforms-inl.h:66-689
//   sigma                    lib/jxl/epf.cc:39-133
//   Gaborish / EPF / XYB     lib/jxl/render_pipeline/stage_{gaborish,epf,xyb}.cc, dec_xyb-inl.h:38-86
//
// This translation unit is compiled with -fmad=false: the compiler never fuses a
// multiply and an add on its own; fmaf() appears exactly where the reference's
// AVX2 path has MulAdd / NegMulAdd, which makes results bit-identical to
// oracle/jxl_oracle.c (rcp_mode 0).
//
// Thread mapping (grids are sized from the device's SM count at run time, 32-wide warps):
//   plan kernel   one CTA (1024 thr) per 256x256 AC group: block-scan of varblock sizes ->
//                 per-block coefficient offsets, per-strategy work lists, sigma plane (one block per thread).
//   8x8 IDCT      idct8_tma_kernel: 8 lanes per block, 4 blocks per warp, coefficients staged one item ahead
//                 with cp.async.bulk + mbarrier (idct8_kernel: the same with ordinary loads).
//   mid IDCT      one warp per "warp item" = 32/W varblocks of one strategy (W = 16, 32 lanes per varblock);
//                 lane = vertical frequency in pass 1, pixel column in pass 2; 1-D transforms live entirely
//                 in registers, one smem transpose in between.
//   large IDCT    64..256 sides: two launches (rows, columns) over slabs of a varblock; 128/256-point
//                 transforms warp-cooperative, column tiles through shared memory.
//   filter        filter_strip_kernel: a CTA owns 256 columns x a row segment and streams the rows through
//                 per-stage rings in shared memory (Gaborish -> EPF0/1/2 -> XYB->RGB -> packing), the EPF
//                 passes on a permutation of the strip's block columns (engaged blocks first).
//                 filter_kernel: generic 64x32 tile + halo version for arbitrary stage masks.
//   upsampling    upsample_kernel: one thread per output pixel, fused with XYB->RGB and the packing.
//   fused         jxl_fused.cuh (opt-in): everything above for the 8x8 class in one persistent kernel.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

// tests/emu compiles this very source for the host (a SIMT emulation shim provides threadIdx,
// __syncthreads, ... ) to check the kernels on a machine without a GPU; inline PTX is the one thing
// that cannot travel, so each use has a host-equivalent behind JXLB_HOST_EMU.  nvcc never defines it.
#ifdef JXLB_HOST_EMU
#define JXLB_PTX 0
#else
#define JXLB_PTX 1
#endif

#define JXT_CONST __device__ __constant__ const
#define JXT_CONST_GMEM __device__ const
#include "jxl_tables.h"
#include "jxl_dc_stage.h"

namespace jxlb {

constexpr float kSqrt2 = 1.41421356237f;  // lib/jxl/dct_scales.h:15
constexpr int kNumStrategies = 27;
constexpr int kFirstLarge = 18;           // strategies >= 18 have a 64+ side

// AcStrategy geometry (lib/jxl/ac_strategy.h:148-173)
__host__ __device__ constexpr int covered_x(int s) {
  constexpr int k[27] = {1, 1, 1, 1, 2, 4, 1, 2, 1, 4, 2, 4, 1, 1, 1, 1, 1, 1, 8, 4, 8, 16, 8, 16, 32, 16, 32};
  return k[s];
}
__host__ __device__ constexpr int covered_y(int s) {
  constexpr int k[27] = {1, 1, 1, 1, 2, 4, 2, 1, 4, 1, 4, 2, 1, 1, 1, 1, 1, 1, 8, 8, 4, 16, 16, 8, 32, 32, 16};
  return k[s];
}

constexpr uint32_t kBmapCopy = 255u;  // bmap kind: pixels come from the XYB planes (varblock not of the 8x8 class)
constexpr uint32_t kBmapSkip = 254u;  // (fused kernel internal: block outside the image)
// strategies whose varblock is one 8x8 block: DCT, IDENTITY, DCT2X2, DCT4X4, DCT4X8, DCT8X4, AFV0..3
__host__ __device__ constexpr bool is_block8_class(int s) { return s <= 3 || (s >= 12 && s <= 17); }

struct FrameDev {
  uint32_t xsize, ysize, xb, yb, xg, yg;
  uint32_t ac_is32;
  uint32_t stage_mask;       // JXLGPU_STAGE_* bits actually run
  uint32_t out_format;
  uint32_t band_y0, band_y1; // pixel rows [band_y0, band_y1) rendered by the filter kernel
  uint32_t out_y0, out_h;    // output addressing: image row stored at output row 0, rows per plane
  // fused all-gather (multi-GPU): every finished pixel is also stored to the same offset of
  // `nrep` peer-mapped buffers over NVLink, or once through an NVSwitch multicast address
  uint32_t nrep;
  char* rep[8];
  char* mc;
  uint32_t need_y0, need_y1; // pixel rows of post-IDCT data the band's filters read (band +- halo)
  uint32_t plan_g0;          // first AC group handled by the plan kernel (band sharding)
  // side info (device)
  const uint8_t* acs;
  const int32_t* quant;
  const uint8_t* sharp;
  const int8_t* ytox;
  const int8_t* ytob;
  uint32_t cmap_stride;
  const float* dc;           // 3 planes [yb][xb]
  const float* dq;           // dequant table
  uint32_t dq_off[3 * kNumStrategies];
  const void* coeff[3];      // channel c of group g starts at coeff[c] + g * coeff_gstride elements
  size_t coeff_gstride;      // 65536 (three planes) or 3*65536 (group-major [g][c][65536])
  // produced by the plan kernel
  uint16_t* coeff_off;       // [yb][xb] offset/64 of the varblock inside its group (first blocks)
  float* sigma;              // [yb][xb] inverse sigma
  uint4* list;               // work lists: {(aby<<16)|abx, coefficient base / 64, raw quant, ytox | ytob<<8}
  uint32_t* counts;          // [27]
  uint32_t list_base[kNumStrategies];
  // fused path (jxl_fused.cuh): one 16-byte record per 8x8 block, [yb][xb]:
  //   {kind (strategy 0..17 of an 8x8-class varblock | kBmapCopy), coefficient base / 64, raw quant, ytox | ytob<<8}
  // and no work lists for the 8x8 class (the fused kernel transforms those itself).
  uint4* bmap;
  uint32_t fused;
  // planes
  float* xyb;                // 3 planes [yb*8][xb*8]
  size_t plane_stride, row_stride;
  // scalars
  float inv_global_scale, quant_scale, x_dm, b_dm;
  float qbias[4];
  float cfl_base_x, cfl_base_b, cfl_scale;
  float gab_w[9];            // normalised: w0,w1,w2 per channel
  float epf_sharp_lut[8];
  float epf_scale[3];
  float epf_quant_mul, epf_sm[3], epf_border_mul;  // epf_sm[pass]: sigma multiplier of pass 0/1/2
  float opsin_m[9], opsin_bias[3], opsin_cbrt[3];
  // upsampling after the filters (stage_upsampling.cc): factor (0/1 = none), output size, the N*N x 25 tap table
  uint32_t ups, out_w, out_hh;
  const float* ups_kernel;
  // noise (stage_noise.cc): three planes [out_hh][out_w] of generator output in [1, 2), the strength LUT
  uint32_t noise;
  const float* noise_planes;
  float noise_lut[8];
  uint32_t skip_xyb;   // frames with upsampling / noise: the strip kernel stops before XYB -> RGB (planar XYB out)
  uint32_t ycbcr;      // colour transform of the frame: 0 = XYB, 1 = YCbCr (kYCbCrStage instead of the opsin inverse)
};

// ---------------------------------------------------------------------------
// mbarrier + bulk async copy (TMA) primitives.  Host emulation (tests/emu): copies are synchronous, the
// barriers around them are the kernel's own __syncthreads().
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) {
#if JXLB_PTX
  return (uint32_t)__cvta_generic_to_shared(p);
#else
  return 0;
#endif
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
#if JXLB_PTX
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#else
  *bar = count;
#endif
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
#if JXLB_PTX
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
#else
  (void)bar; (void)bytes;
#endif
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#if JXLB_PTX
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
#else
  (void)bar; (void)parity;
  __syncwarp();  // (emulation: the copies were made synchronously by other lanes of this warp, or before a barrier)
#endif
}
// global -> shared, completion counted in bytes on `bar` (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
#if JXLB_PTX
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_addr(dst_smem)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
#else
  memcpy(dst_smem, src, bytes);
  (void)bar;
#endif
}
// shared -> global (bulk group of the issuing thread)
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src_smem, uint32_t bytes) {
#if JXLB_PTX
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_addr(src_smem)), "r"(bytes) : "memory");
#else
  memcpy(dst, src_smem, bytes);
#endif
}
__device__ __forceinline__ void bulk_commit() {
#if JXLB_PTX
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void bulk_wait_read_all() {  // the sources of all committed groups have been read
#if JXLB_PTX
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
#endif
}
__device__ __forceinline__ void bulk_wait_all() {
#if JXLB_PTX
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
#endif
}
// 16 bytes global -> shared without a register on the way (cp.async, completion per thread in commit groups)
__device__ __forceinline__ void async_copy16(void* dst_smem, const void* src) {
#if JXLB_PTX
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_addr(dst_smem)), "l"(src) : "memory");
#else
  memcpy(dst_smem, src, 16);
#endif
}
__device__ __forceinline__ void async_commit() {
#if JXLB_PTX
  asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
template <int N>  // all but the N most recent commit groups of this thread have landed
__device__ __forceinline__ void async_wait() {
#if JXLB_PTX
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
#endif
}
// 16-byte global store with an L2 evict_last hint (st.global.L2::cache_hint).  The 8x8 IDCT stores its XYB
// rows in 32-byte pieces that the filter kernel reads next; kept in L2 ahead of the streamed coefficients,
// they make idct8_tma_kernel about 6 % faster on H100 (DESIGN.md §4).
__device__ __forceinline__ void st_global_l2_keep(float* p, float4 v) {
#if JXLB_PTX
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w), "l"(pol) : "memory");
#else
  *reinterpret_cast<float4*>(p) = v;
#endif
}
// generic-proxy writes to shared memory -> visible to the async proxy (the TMA unit)
__device__ __forceinline__ void fence_async_smem() {
#if JXLB_PTX
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}

// ---------------------------------------------------------------------------
// 1-D transforms in registers
// ---------------------------------------------------------------------------
// IDCT1DImpl<N> (dct-inl.h:191-232): even/odd split, BTranspose, butterflies.
template <int N>
__device__ __forceinline__ void idct1d(float* v) {
  if constexpr (N == 1) {
    return;
  } else if constexpr (N == 2) {
    const float a = v[0], b = v[1];
    v[0] = a + b;
    v[1] = a - b;
  } else {
    constexpr int H = N / 2;
    float e[H], o[H];
#pragma unroll
    for (int i = 0; i < H; i++) { e[i] = v[2 * i]; o[i] = v[2 * i + 1]; }
    idct1d<H>(e);
#pragma unroll
    for (int i = H - 1; i > 0; i--) o[i] = o[i] + o[i - 1];
    o[0] = o[0] * kSqrt2;
    idct1d<H>(o);
#pragma unroll
    for (int i = 0; i < H; i++) {
      const float w = JXT_WC[H - 2 + i];
      v[i] = fmaf(w, o[i], e[i]);
      v[N - 1 - i] = fmaf(-w, o[i], e[i]);
    }
  }
}

// DCT1DImpl<N> (dct-inl.h:158-189), unscaled.
template <int N>
__device__ __forceinline__ void dct1d(float* v) {
  if constexpr (N == 1) {
    return;
  } else if constexpr (N == 2) {
    const float a = v[0], b = v[1];
    v[0] = a + b;
    v[1] = a - b;
  } else {
    constexpr int H = N / 2;
    float t0[H], t1[H];
#pragma unroll
    for (int i = 0; i < H; i++) t0[i] = v[i] + v[N - 1 - i];
    dct1d<H>(t0);
#pragma unroll
    for (int i = 0; i < H; i++) t1[i] = (v[i] - v[N - 1 - i]) * JXT_WC[H - 2 + i];
    dct1d<H>(t1);
    t1[0] = fmaf(t1[0], kSqrt2, t1[1]);
#pragma unroll
    for (int i = 1; i + 1 < H; i++) t1[i] = t1[i] + t1[i + 1];
#pragma unroll
    for (int i = 0; i < H; i++) { v[2 * i] = t0[i]; v[2 * i + 1] = t1[i]; }
  }
}

// ---------------------------------------------------------------------------
// dequantisation (dec_group.cc:115-181, quantizer-inl.h:35-67)
// ---------------------------------------------------------------------------
// Correctly rounded 1/x for the dequantiser: MUFU.RCP + one FMA Newton step equals __frcp_rn(x)
// for every integer 2 <= |x| < 2^24 (exhaustive check: tools/probe/rcp_probe.cu).
// [2^23, 2^24) contains every 24-bit significand, MUFU.RCP and FMA are exponent-invariant for
// normal numbers, and 1/x stays normal for |x| <= 2^31, so the identity holds for every int32
// coefficient; no special-case branch is needed.  (x = 0 yields NaN, which callers discard.)
__device__ __forceinline__ float rcp_int(float x) {
#if JXLB_PTX
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  const float e = fmaf(-x, r, 1.0f);
  return fmaf(r, e, r);
#else
  return 1.0f / x;  // the correctly rounded reciprocal, which is what the sequence above yields
#endif
}

// AdjustQuantBias (quantizer-inl.h:35-67), branch-free: q in {-1,0,1} -> q*biases[c] (exact),
// otherwise q - biases[3] * (1/q) as one FMA.
__device__ __forceinline__ float adjust_quant_bias(int q, float bias_c, float bias3) {
  const float fq = (float)q;
  const float small = bias_c * fq;
  const float big = fmaf(-bias3, rcp_int(fq), fq);
  return fabsf(fq) < 1.125f ? small : big;
}

template <bool I32>
__device__ __forceinline__ int load_q(const void* p, size_t i) {
  if constexpr (I32) return __ldg(reinterpret_cast<const int32_t*>(p) + i);
  else return (int)__ldg(reinterpret_cast<const int16_t*>(p) + i);
}

struct VarblockCtx {
  uint32_t abx, aby;
  size_t cbase;      // element index of coefficient 0 in the channel plane
  float sx, sy, sb;  // scaled dequant multipliers
  float x_cc, b_cc;
};

__device__ __forceinline__ VarblockCtx make_ctx(const FrameDev& P, uint4 entry) {
  VarblockCtx v;
  v.abx = entry.x & 0xffffu;
  v.aby = entry.x >> 16;
  v.cbase = (size_t)entry.y * 64u;
  const float s = P.inv_global_scale / (float)(int)entry.z;
  v.sx = s * P.x_dm;
  v.sy = s;
  v.sb = s * P.b_dm;
  v.x_cc = P.cfl_base_x + (float)(int)(int8_t)(entry.w & 0xffu) * P.cfl_scale;
  v.b_cc = P.cfl_base_b + (float)(int)(int8_t)((entry.w >> 8) & 0xffu) * P.cfl_scale;
  return v;
}

// dequantised coefficient i (index inside the varblock) of channel c
template <bool I32>
__device__ __forceinline__ float dequant(const FrameDev& P, const VarblockCtx& v, int kind, int c,
                                         uint32_t i) {
  const int qy = load_q<I32>(P.coeff[1], v.cbase + i);
  const float y_mul = __ldg(P.dq + P.dq_off[3 * kind + 1] + i) * v.sy;
  const float dy = adjust_quant_bias(qy, P.qbias[1], P.qbias[3]) * y_mul;
  if (c == 1) return dy;
  const int qc = load_q<I32>(P.coeff[c], v.cbase + i);
  const float c_mul = __ldg(P.dq + P.dq_off[3 * kind + c] + i) * (c == 0 ? v.sx : v.sb);
  const float dc_ = adjust_quant_bias(qc, P.qbias[c], P.qbias[3]) * c_mul;
  return fmaf(c == 0 ? v.x_cc : v.b_cc, dy, dc_);
}

// ---------------------------------------------------------------------------
// plan kernel: one CTA (1024 threads) per AC group
// ---------------------------------------------------------------------------
#ifndef JXLB_STRIP_TU  // (the strip translation units compile the row-streaming filter kernel only)
__global__ void __launch_bounds__(1024) plan_kernel(const __grid_constant__ FrameDev P, int want_sigma) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t local_count[kNumStrategies];
  __shared__ uint32_t local_base[kNumStrategies];
  __shared__ uint16_t owner[1024];
  const uint32_t t = threadIdx.x;
  const uint32_t g = blockIdx.x + P.plan_g0;
  const uint32_t gx = g % P.xg, gy = g / P.xg;
  const uint32_t abx = gx * 32 + (t & 31), aby = gy * 32 + (t >> 5);
  const bool valid = abx < P.xb && aby < P.yb;
  if (t < kNumStrategies) local_count[t] = 0;
  const size_t bi = (size_t)aby * P.xb + abx;
  const uint32_t raw = valid ? P.acs[bi] : 0u;
  const bool first = valid && (raw & 1u);
  const int s = min((int)(raw >> 1), kNumStrategies - 1);  // (a corrupt strategy byte must not index past the tables)
  const uint32_t area = first ? (uint32_t)(covered_x(s) * covered_y(s)) : 0u;
  // exclusive scan of `area` in raster order (dec_group.cc:221,335-359: running offset)
  uint32_t incl = area;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t n = __shfl_up_sync(0xffffffffu, incl, d);
    if ((t & 31) >= (uint32_t)d) incl += n;
  }
  if ((t & 31) == 31) warp_sums[t >> 5] = incl;
  __syncthreads();
  if (t < 32) {
    uint32_t w = warp_sums[t];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t n = __shfl_up_sync(0xffffffffu, w, d);
      if (t >= (uint32_t)d) w += n;
    }
    warp_sums[t] = w;
  }
  __syncthreads();
  const uint32_t off = incl - area + ((t >> 5) ? warp_sums[(t >> 5) - 1] : 0u);
  uint32_t rank = 0;
  // band sharding: only varblocks that intersect the rows this band's filters read are listed
  bool wanted = first && (aby * 8u < P.need_y1) && ((aby + (uint32_t)covered_y(s)) * 8u > P.need_y0);
  if (first) P.coeff_off[bi] = (uint16_t)off;
  const bool inline8 = P.fused && is_block8_class(s);
  if (P.fused && valid) {
    // fused path: the 8x8 class is transformed by the fused kernel straight from this record; every other
    // block is fetched from the XYB planes the mid / large kernels fill (kBmapCopy)
    uint4 rec = make_uint4(kBmapCopy, 0u, 1u, 0u);
    if (first && inline8) {
      const size_t ti = (size_t)(aby >> 3) * P.cmap_stride + (abx >> 3);
      rec = make_uint4((uint32_t)s, (uint32_t)((size_t)g * (P.coeff_gstride >> 6) + off), (uint32_t)P.quant[bi],
                       (uint32_t)(uint8_t)P.ytox[ti] | ((uint32_t)(uint8_t)P.ytob[ti] << 8));
    }
    P.bmap[bi] = rec;
  }
  const bool listed = wanted && !inline8;
  if (listed) rank = atomicAdd(&local_count[s], 1u);
  __syncthreads();
  if (t < kNumStrategies && local_count[t]) local_base[t] = atomicAdd(&P.counts[t], local_count[t]);
  __syncthreads();
  if (wanted) {
    // everything an IDCT warp needs about the varblock in one 16-byte record (one load instead of
    // a dependent chain list -> coeff_off / quant / cmap)
    if (listed) {
      const size_t ti = (size_t)(aby >> 3) * P.cmap_stride + (abx >> 3);
      const uint32_t cfl = (uint32_t)(uint8_t)P.ytox[ti] | ((uint32_t)(uint8_t)P.ytob[ti] << 8);
      P.list[P.list_base[s] + local_base[s] + rank] =
          make_uint4((aby << 16) | abx, (uint32_t)((size_t)g * (P.coeff_gstride >> 6) + off), (uint32_t)P.quant[bi], cfl);
    }
  }
  if (want_sigma) {
    // ComputeSigma (epf.cc:39-133): every block of a varblock takes the quantiser of the varblock's first
    // block and its own sharpness.  The first block's thread only marks the blocks it covers (shared-memory
    // stores); the divisions and global accesses are then done by all 1024 threads, one block each -- a
    // 256x256 varblock used to leave one thread looping over 1024 blocks.
    owner[t] = (uint16_t)t;
    __syncthreads();
    if (first) {
      const int ny = min(covered_y(s), 32 - (int)(t >> 5)), nx = min(covered_x(s), 32 - (int)(t & 31));  // (never past the group)
      for (int iy = 0; iy < ny; iy++)
        for (int ix = 0; ix < nx; ix++) owner[t + iy * 32 + ix] = (uint16_t)t;
    }
    __syncthreads();
    if (valid) {
      const uint32_t o = owner[t];
      const size_t bo = (size_t)(gy * 32 + (o >> 5)) * P.xb + gx * 32 + (o & 31);
      const float kInvSigmaNum = -1.1715728752538099024f;
      const float sigma_quant = P.epf_quant_mul / (P.quant_scale * (float)P.quant[bo] * kInvSigmaNum);
      float sg = sigma_quant * P.epf_sharp_lut[P.sharp[bi]];
      sg = fminf(-1e-4f, sg);
      P.sigma[bi] = 1.0f / sg;
    }
  }
}

#endif  // JXLB_STRIP_TU

// ---------------------------------------------------------------------------
// LLF from DC for multi-block DCTs (dec_transforms-inl.h:35-64): forward
// cy x cx DCT of the DC window, rescaled. Cooperative: `nl` lanes/threads with
// index l; t0/out are shared scratch of cy*cx floats; sync() separates phases.
// Result: out[j*cx + k] = LLF value of (vertical freq j, horizontal freq k).
// ---------------------------------------------------------------------------
template <int CY, int CX, typename Sync>
__device__ __forceinline__ void llf_from_dc(const float* dc, size_t dc_stride, int l, float* t0,
                                            float* out, Sync sync) {
  if (l < CX) {
    float col[CY];
#pragma unroll
    for (int y = 0; y < CY; y++) col[y] = __ldg(dc + (size_t)y * dc_stride + l);
    dct1d<CY>(col);
#pragma unroll
    for (int y = 0; y < CY; y++) t0[y * CX + l] = (1.0f / CY) * col[y];
  }
  sync();
  if (l < CY) {
    float row[CX];
#pragma unroll
    for (int x = 0; x < CX; x++) row[x] = t0[l * CX + x];
    dct1d<CX>(row);
    const float sy = JXT_RESAMPLE[CY - 1 + l];
#pragma unroll
    for (int x = 0; x < CX; x++) {
      const float v = (1.0f / CX) * row[x];
      const float sx = JXT_RESAMPLE[CX - 1 + x];
      // multiplication order of ReinterpretingDCT: first-index scale first
      out[l * CX + x] = (CY < CX) ? (v * sy) * sx : (v * sx) * sy;
    }
  }
  sync();
}

struct WarpSync {
  __device__ __forceinline__ void operator()() const { __syncwarp(); }
};
struct BlockSync {
  __device__ __forceinline__ void operator()() const { __syncthreads(); }
};

// ---------------------------------------------------------------------------
// small IDCT: plain DCTs with R, C <= 32 (ComputeScaledIDCT<R,C>, dct-inl.h:376-397)
// W = max(R,C) lanes per varblock. sm: per-warp scratch (>= 32/W * (R*(C+1) + 2*CY*CX) floats).
// ---------------------------------------------------------------------------
template <int R, int C, bool I32>
__device__ __forceinline__ void small_dct_item(const FrameDev& P, int kind, uint32_t first_entry_idx,
                                               uint32_t count, float* sm) {
  constexpr int W = R > C ? R : C;
  constexpr int SLOTS = 32 / W;
  constexpr int CY = R / 8, CX = C / 8;
  constexpr int TS = R * (C + 1);             // transpose buffer per slot
  constexpr int SLOT_FLOATS = TS + 2 * CY * CX;
  const int lane = threadIdx.x & 31;
  const int slot = lane / W, l = lane % W;
  const uint32_t eidx = first_entry_idx + slot;
  const bool active = eidx < count;
  float* T = sm + slot * SLOT_FLOATS;
  float* llf = T + TS;
  float* llf_tmp = llf + CY * CX;
  VarblockCtx vb;
  if (active) vb = make_ctx(P, __ldg(P.list + P.list_base[kind] + eidx));
  else vb = VarblockCtx{};
#pragma unroll 1
  for (int c = 0; c < 3; c++) {
    // ---- LLF (cooperative inside the slot) ----
    if constexpr (CY * CX > 1) {
      const float* dcp = P.dc + (size_t)c * P.yb * P.xb + (active ? (size_t)vb.aby * P.xb + vb.abx : 0);
      llf_from_dc<CY, CX>(dcp, P.xb, active ? l : 1000, llf_tmp, llf, WarpSync());
    }
    // ---- pass 1: lane j = vertical frequency, IDCT over horizontal frequency k ----
    float v[C];
    if (active && l < R) {
#pragma unroll
      for (int k = 0; k < C; k++) {
        const uint32_t i = (R >= C) ? (uint32_t)(k * R + l) : (uint32_t)(l * C + k);
        v[k] = dequant<I32>(P, vb, kind, c, i);
      }
      if constexpr (CY * CX > 1) {
        if (l < CY) {
#pragma unroll
          for (int k = 0; k < CX; k++) v[k] = llf[l * CX + k];
        }
      } else {
        if (l == 0) v[0] = __ldg(P.dc + (size_t)c * P.yb * P.xb + (size_t)vb.aby * P.xb + vb.abx);
      }
      idct1d<C>(v);
#pragma unroll
      for (int x = 0; x < C; x++) T[l * (C + 1) + x] = v[x];
    }
    __syncwarp();
    // ---- pass 2: lane x = pixel column, IDCT over vertical frequency ----
    if (active && l < C) {
      float u[R];
#pragma unroll
      for (int j = 0; j < R; j++) u[j] = T[j * (C + 1) + l];
      idct1d<R>(u);
      float* out = P.xyb + (size_t)c * P.plane_stride + (size_t)vb.aby * 8 * P.row_stride + vb.abx * 8 + l;
#pragma unroll
      for (int y = 0; y < R; y++) out[(size_t)y * P.row_stride] = u[y];
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------
// small IDCT: the 8x8 specials (dec_transforms-inl.h:66-93,399-581). 8 lanes per block,
// 4 blocks per warp. Per slot scratch: co[64] coefficients, tmp[64], px[64] pixels.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void hadamard4(float b00, float b01, float b10, float b11, float* dcs) {
  dcs[0] = b00 + b01 + b10 + b11;
  dcs[1] = b00 + b01 - b10 - b11;
  dcs[2] = b00 - b01 + b10 - b11;
  dcs[3] = b00 - b01 - b10 + b11;
}

// One row (8 consecutive coefficients) of a channel plane as integers.
template <bool I32>
__device__ __forceinline__ void load_row8(const void* plane, size_t elem, int* q) {
  if constexpr (I32) {
    const int4* p = reinterpret_cast<const int4*>(reinterpret_cast<const int32_t*>(plane) + elem);
    const int4 a = __ldg(p), b = __ldg(p + 1);
    q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
  } else {
    const int4 a = __ldg(reinterpret_cast<const int4*>(reinterpret_cast<const int16_t*>(plane) + elem));
    const int w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      q[2 * i] = (int)(short)(w[i] & 0xffff);
      q[2 * i + 1] = w[i] >> 16;
    }
  }
}

__device__ __forceinline__ void load_row8f(const float* p, float* m) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  m[0] = a.x; m[1] = a.y; m[2] = a.z; m[3] = a.w; m[4] = b.x; m[5] = b.y; m[6] = b.z; m[7] = b.w;
}
// row l of an 8x8 float matrix in SHARED memory (same bank-conflict-free half order as load_row8_smem)
__device__ __forceinline__ void load_row8f_smem(const float* mat, int l, float* m) {
  const float4* p = reinterpret_cast<const float4*>(mat + l * 8);
  const int sw = (l >> 2) & 1;
  const float4 u = p[sw], v = p[sw ^ 1];
  const float4 a = sw ? v : u, b = sw ? u : v;
  m[0] = a.x; m[1] = a.y; m[2] = a.z; m[3] = a.w; m[4] = b.x; m[5] = b.y; m[6] = b.z; m[7] = b.w;
}

// One row (8 consecutive coefficients) of a block held in SHARED memory (the fused kernel's staging).
template <bool I32>
__device__ __forceinline__ void load_row8_smem(const void* block, int elem, int* q) {
  if constexpr (I32) {
    // eight lanes read eight 32-byte rows with two 16-byte loads each: rows 4..7 take their second half first,
    // so that the eight lanes of a load phase touch all 32 banks once instead of 16 banks twice
    const int4* p = reinterpret_cast<const int4*>(reinterpret_cast<const int32_t*>(block) + elem);
    const int sw = (elem >> 5) & 1;
    const int4 u = p[sw], v = p[sw ^ 1];
    const int4 a = sw ? v : u, b = sw ? u : v;
    q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
  } else {
    const int4 a = *reinterpret_cast<const int4*>(reinterpret_cast<const int16_t*>(block) + elem);
    const int w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      q[2 * i] = (int)(short)(w[i] & 0xffff);
      q[2 * i + 1] = w[i] >> 16;
    }
  }
}

// The 8 coefficients lane l of an 8x8-class block owns in one channel: column l for DCT8x8 (`col`: its first
// 1-D pass runs down the columns in registers), row l for the specials.
//   load_lane8: from the channel plane in HBM (e0 = element index of coefficient 0); a row is two / one 16-byte
//     loads when the plane is 16-byte aligned (`vec`), element loads otherwise
//   load_lane8_smem: from the block staged in SHARED memory
template <bool I32>
__device__ __forceinline__ void load_lane8(const void* plane, size_t e0, int l, bool col, bool vec, int* q) {
  if (col) {
#pragma unroll
    for (int k = 0; k < 8; k++) q[k] = load_q<I32>(plane, e0 + k * 8 + l);
  } else if (vec) {
    load_row8<I32>(plane, e0 + (size_t)l * 8, q);
  } else {
#pragma unroll
    for (int k = 0; k < 8; k++) q[k] = load_q<I32>(plane, e0 + (size_t)l * 8 + k);
  }
}
template <bool I32>
__device__ __forceinline__ void load_lane8_smem(const void* block, int l, bool col, int* q) {
  if (col) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
      if constexpr (I32) q[k] = reinterpret_cast<const int32_t*>(block)[k * 8 + l];
      else q[k] = reinterpret_cast<const int16_t*>(block)[k * 8 + l];
    }
  } else {
    load_row8_smem<I32>(block, l * 8, q);
  }
}

// Dequantisation of lane l's 8 coefficients of an 8x8-class block (column l if `col`, else row l; see
// load_lane8), all three channels (dec_group.cc:115-181), one channel after the other: Y first, CfL adds
// it to X and B.  load_q(c, q) fills the 8 integers of channel c.
//   dqx/dqy/dqb: the strategy's 8x8 dequant matrices (global memory, or a shared-memory copy)
// Coefficient (0, 0), which lane 0 holds in either layout, is replaced by the DC afterwards (block8_dc).
template <bool SMEM, class LoadQ>
__device__ __forceinline__ void block8_dequant_m(const FrameDev& P, const float* dqx, const float* dqy,
                                                 const float* dqb, const VarblockCtx& vb, int l, bool col,
                                                 const LoadQ& load_q, float (&val)[3][8]) {
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const int c = i == 0 ? 1 : (i == 1 ? 0 : 2);
    const float* dqc = c == 0 ? dqx : (c == 1 ? dqy : dqb);
    const float s = c == 0 ? vb.sx : (c == 1 ? vb.sy : vb.sb);
    int q[8];
    float m[8];
    load_q(c, q);
    if (col) {
#pragma unroll
      for (int k = 0; k < 8; k++) {
        if constexpr (SMEM) m[k] = dqc[k * 8 + l];
        else m[k] = __ldg(dqc + k * 8 + l);
      }
    } else if constexpr (SMEM) {
      load_row8f_smem(dqc, l, m);
    } else {
      load_row8f(dqc + l * 8, m);
    }
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const float d = adjust_quant_bias(q[e], P.qbias[c], P.qbias[3]) * (m[e] * s);
      val[c][e] = c == 1 ? d : fmaf(c == 0 ? vb.x_cc : vb.b_cc, val[1][e], d);
    }
  }
}

// LowestFrequenciesFromDC for the 8x8 class: llf[0] = dc[0], in lane 0
__device__ __forceinline__ void block8_dc(const FrameDev& P, const VarblockCtx& vb, int l, float (&val)[3][8]) {
  if (l == 0) {
    const size_t bi = (size_t)vb.aby * P.xb + vb.abx;
#pragma unroll
    for (int c = 0; c < 3; c++) val[c][0] = __ldg(P.dc + (size_t)c * P.yb * P.xb + bi);
  }
}

template <class LoadQ>
__device__ __forceinline__ void block8_dequant(const FrameDev& P, int dqkind, const VarblockCtx& vb, int l, bool col,
                                               const LoadQ& load_q, float (&val)[3][8]) {
  block8_dequant_m<false>(P, P.dq + P.dq_off[3 * dqkind + 0], P.dq + P.dq_off[3 * dqkind + 1],
                          P.dq + P.dq_off[3 * dqkind + 2], vb, l, col, load_q, val);
  block8_dc(P, vb, l, val);
}

// Where the pixels of an 8x8-class block go.
//   Block8ToPlanes: the XYB planes in HBM (idct8_kernel).  The specials assemble the block in a 64-float
//     scratch (row pitch 8) and lane l stores pixel row l with two 16-byte stores.
//   (the fused kernel's policy, Block8ToRing in jxl_fused.cuh, writes straight into its shared-memory
//     pixel ring: row pitch = one ring row.)
// Interface: kPitch; px(c) = where pixel (y, x) of channel c is assembled (px(c)[y * kPitch + x]);
// a plain DCT8x8 leaves either through dct_col(c, l, u, active) = column l (kDctRows false), or, with kDctRows,
// assembled in shared memory (8 rows at pitch 8) through dct_rows(c, l, px, active); no barrier in either;
// finish(c, l, active) after the specials.
struct Block8ToPlanes {
  static constexpr int kPitch = 8;
  static constexpr bool kGuardPx = false;  // inactive slots assemble garbage in their own scratch
  static constexpr bool kDctRows = true;
  float* scratch;
  float* plane0;  // channel 0, pixel (0, 0) of the block
  size_t plane_stride, row_stride;
  __device__ __forceinline__ float* px(int) const { return scratch; }
  // lane l stores the half (l & 1) of rows (l >> 1) and (l >> 1) + 4: each 16-byte store instruction of a warp
  // writes four whole 32-byte rows per block (column stores take eight instructions per channel)
  __device__ __forceinline__ void dct_rows(int c, int l, const float* px, bool active) const {
    if (active) {
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const int y = (l >> 1) + 4 * k, h = (l & 1) * 4;
        const float4 a = *reinterpret_cast<const float4*>(px + y * 8 + h);
        st_global_l2_keep(plane0 + (size_t)c * plane_stride + (size_t)y * row_stride + h, a);
      }
    }
  }
  __device__ __forceinline__ void finish(int c, int l, bool active) const {
    __syncwarp();
    if (active) {  // lane l stores pixel row l (2 x 16 B)
      float* out = plane0 + (size_t)c * plane_stride + (size_t)l * row_stride;
      const float4 a = *reinterpret_cast<const float4*>(scratch + l * 8);
      const float4 b = *reinterpret_cast<const float4*>(scratch + l * 8 + 4);
      st_global_l2_keep(out, a);
      st_global_l2_keep(out + 4, b);
    }
    __syncwarp();
  }
};

// The 2-D inverse transform of one 8x8-class block per 8-lane slot (4 slots per warp), from the
// dequantised coefficients val[c][e] to pixels, for strategy `kind` -- the same for the whole warp.  Lane l
// holds coefficient column l for DCT8x8 and coefficient row l for the specials (load_lane8).  Slots with
// active == false run the same instruction stream (every __syncwarp() is reached by all 32 lanes) but store
// nothing outside their scratch.
// scr: 192 floats of per-slot scratch (the specials: coefficients at scr, their 1-D pass at scr + 64).
template <class Out>
__device__ __forceinline__ void block8_transform(int kind, bool active, const float (&val)[3][8], int l,
                                                 float* scr, const Out& out) {
  constexpr int PP = Out::kPitch;
#define JXLB_PX_OK (!Out::kGuardPx || active)
  if (kind == 0) {
    // ---- DCT 8x8: ComputeScaledIDCT<8,8> (dct-inl.h:376-397) ----
    // pass 1 over the vertical frequency k, in registers (lane l = column l); the three channels' results
    // go through scr as rows (channel c at scr + 64c, pitch 8, the halves of rows 4..7 swapped so that the
    // 16-byte stores of the eight lanes hit all 32 banks once); one barrier; pass 2, lane l = pixel column l
#pragma unroll
    for (int c = 0; c < 3; c++) {
      float v[8];
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] = val[c][k];
      idct1d<8>(v);
      float* row = scr + c * 64 + l * 8;
      const int sw = l & 4;
      *reinterpret_cast<float4*>(row + sw) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(row + (sw ^ 4)) = make_float4(v[4], v[5], v[6], v[7]);
    }
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 3; c++) {
      float u[8];
#pragma unroll
      for (int j = 0; j < 8; j++) u[j] = scr[c * 64 + j * 8 + (l ^ (j & 4))];
      idct1d<8>(u);
      if constexpr (Out::kDctRows) {
        __syncwarp();  // channel c's pass-1 rows are read: its pixels take their place (row y at scr + 64c + 8y)
#pragma unroll
        for (int y = 0; y < 8; y++) scr[c * 64 + y * 8 + l] = u[y];
      } else {
        out.dct_col(c, l, u, active);
      }
    }
    __syncwarp();
    if constexpr (Out::kDctRows) {
#pragma unroll
      for (int c = 0; c < 3; c++) out.dct_rows(c, l, scr + c * 64, active);
      __syncwarp();
    }
    return;  // scr is free again
  }
  float* co = scr;
  float* tmp = scr + 64;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float* px = out.px(c);
    *reinterpret_cast<float4*>(co + l * 8) = make_float4(val[c][0], val[c][1], val[c][2], val[c][3]);
    *reinterpret_cast<float4*>(co + l * 8 + 4) = make_float4(val[c][4], val[c][5], val[c][6], val[c][7]);
    __syncwarp();
    {
      switch (kind) {
        case 1: {  // IDENTITY (dec_transforms-inl.h:463-499)
          if (l < 4) {
            const int y = l >> 1, x = l & 1;
            float dcs[4];
            hadamard4(co[0], co[1], co[8], co[9], dcs);
            const float block_dc = dcs[y * 2 + x];
            float residual_sum = 0.0f;
#pragma unroll
            for (int iy = 0; iy < 4; iy++)
#pragma unroll
              for (int ix = 0; ix < 4; ix++) {
                if (ix == 0 && iy == 0) continue;
                residual_sum += co[(y + iy * 2) * 8 + x + ix * 2];
              }
            const float p11 = block_dc - residual_sum * (1.0f / 16);
            if (JXLB_PX_OK) {
#pragma unroll
              for (int iy = 0; iy < 4; iy++)
#pragma unroll
                for (int ix = 0; ix < 4; ix++) {
                  if (ix == 1 && iy == 1) continue;
                  px[(y * 4 + iy) * PP + x * 4 + ix] = co[(y + iy * 2) * 8 + x + ix * 2] + p11;
                }
              px[(4 * y + 1) * PP + 4 * x + 1] = p11;
              px[(y * 4) * PP + x * 4] = co[(y + 2) * 8 + x + 2] + p11;
            }
          }
          break;
        }
        case 2: {  // DCT2X2 (569-581): IDCT2TopBlock<2>, <4>, <8> in place
#pragma unroll
          for (int S = 2; S <= 8; S *= 2) {
            const int n = S / 2;
            float r[2][4];
#pragma unroll
            for (int it = 0; it < 2; it++) {
              const int item = l + it * 8;
              if (item < n * n) {
                const int y = item / n, x = item % n;
                const float c00 = co[y * 8 + x], c01 = co[y * 8 + n + x];
                const float c10 = co[(y + n) * 8 + x], c11 = co[(y + n) * 8 + n + x];
                r[it][0] = c00 + c01 + c10 + c11;
                r[it][1] = c00 + c01 - c10 - c11;
                r[it][2] = c00 - c01 + c10 - c11;
                r[it][3] = c00 - c01 - c10 + c11;
              }
            }
            __syncwarp();
#pragma unroll
            for (int it = 0; it < 2; it++) {
              const int item = l + it * 8;
              if (item < n * n) {
                const int y = item / n, x = item % n;
                if (S == 8) {
                  if (JXLB_PX_OK) {
                    px[(y * 2) * PP + x * 2] = r[it][0];
                    px[(y * 2) * PP + x * 2 + 1] = r[it][1];
                    px[(y * 2 + 1) * PP + x * 2] = r[it][2];
                    px[(y * 2 + 1) * PP + x * 2 + 1] = r[it][3];
                  }
                } else {
                  co[(y * 2) * 8 + x * 2] = r[it][0];
                  co[(y * 2) * 8 + x * 2 + 1] = r[it][1];
                  co[(y * 2 + 1) * 8 + x * 2] = r[it][2];
                  co[(y * 2 + 1) * 8 + x * 2 + 1] = r[it][3];
                }
              }
            }
            __syncwarp();
          }
          break;
        }
        case 3: {  // DCT4X4 (541-568)
          float dcs[4];
          hadamard4(co[0], co[1], co[8], co[9], dcs);
#pragma unroll
          for (int it = 0; it < 2; it++) {  // pass 1: (sub-block, j)
            const int sub = (l >> 2) + 2 * it, j = l & 3;
            const int y = sub >> 1, x = sub & 1;
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) v[k] = co[(y + k * 2) * 8 + x + j * 2];
            if (j == 0) v[0] = dcs[sub];
            idct1d<4>(v);
#pragma unroll
            for (int xx = 0; xx < 4; xx++) tmp[sub * 16 + j * 4 + xx] = v[xx];
          }
          __syncwarp();
#pragma unroll
          for (int it = 0; it < 2; it++) {  // pass 2: (sub-block, column)
            const int sub = (l >> 2) + 2 * it, xx = l & 3;
            const int y = sub >> 1, x = sub & 1;
            float u[4];
#pragma unroll
            for (int j = 0; j < 4; j++) u[j] = tmp[sub * 16 + j * 4 + xx];
            idct1d<4>(u);
            if (JXLB_PX_OK) {
#pragma unroll
              for (int yy = 0; yy < 4; yy++) px[(4 * y + yy) * PP + 4 * x + xx] = u[yy];
            }
          }
          break;
        }
        case 12: {  // DCT4X8 (520-540): two 4-row halves
          const float b0 = co[0], b1 = co[8];
          {
            const int half = l >> 2, j = l & 3;
            float v[8];
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] = co[(half + j * 2) * 8 + k];
            if (j == 0) v[0] = half ? (b0 - b1) : (b0 + b1);
            idct1d<8>(v);
#pragma unroll
            for (int x = 0; x < 8; x++) tmp[half * 32 + j * 8 + x] = v[x];
          }
          __syncwarp();
#pragma unroll
          for (int half = 0; half < 2; half++) {
            float u[4];
#pragma unroll
            for (int j = 0; j < 4; j++) u[j] = tmp[half * 32 + j * 8 + l];
            idct1d<4>(u);
            if (JXLB_PX_OK) {
#pragma unroll
              for (int yy = 0; yy < 4; yy++) px[(4 * half + yy) * PP + l] = u[yy];
            }
          }
          break;
        }
        case 13: {  // DCT8X4 (500-519): two 4-column halves
          const float b0 = co[0], b1 = co[8];
#pragma unroll
          for (int half = 0; half < 2; half++) {
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) v[k] = co[(half + k * 2) * 8 + l];
            if (l == 0) v[0] = half ? (b0 - b1) : (b0 + b1);
            idct1d<4>(v);
#pragma unroll
            for (int xx = 0; xx < 4; xx++) tmp[half * 32 + l * 4 + xx] = v[xx];
          }
          __syncwarp();
          {
            const int half = l >> 2, xx = l & 3;
            float u[8];
#pragma unroll
            for (int j = 0; j < 8; j++) u[j] = tmp[half * 32 + j * 4 + xx];
            idct1d<8>(u);
            if (JXLB_PX_OK) {
#pragma unroll
              for (int yy = 0; yy < 8; yy++) px[yy * PP + half * 4 + xx] = u[yy];
            }
          }
          break;
        }
        default: {  // AFV0..3 (399-454)
          const int afv_kind = kind - 14;
          const int afv_x = afv_kind & 1, afv_y = afv_kind >> 1;
          const float b00 = co[0], b01 = co[1], b10 = co[8];
          const float dcs0 = (b00 + b10 + b01) * 4.0f;
          const float dcs1 = (b00 + b10 - b01);
          const float dcs2 = b00 - b10;
          // (a) AFVIDCT4x4: two of the 16 outputs per lane
#pragma unroll
          for (int it = 0; it < 2; it++) {
            const int i = l + 8 * it;
            float p = 0.0f;
#pragma unroll
            for (int j = 0; j < 16; j++) {
              const float cf = (j == 0) ? dcs0 : co[(j >> 2) * 2 * 8 + (j & 3) * 2];
              p = fmaf(cf, JXT_AFV_BASIS[j][i], p);
            }
            const int r = i >> 2, cc = i & 3;
            const int iy = afv_y ? 3 - r : r, ix = afv_x ? 3 - cc : cc;
            if (JXLB_PX_OK) px[(iy + afv_y * 4) * PP + afv_x * 4 + ix] = p;
          }
          // (b) 4x4 IDCT of the (odd column) interleave, (c) 4x8 IDCT of the odd rows: pass 1
          if (l < 4) {
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) v[k] = co[k * 2 * 8 + l * 2 + 1];
            if (l == 0) v[0] = dcs1;
            idct1d<4>(v);
#pragma unroll
            for (int xx = 0; xx < 4; xx++) tmp[l * 4 + xx] = v[xx];
          } else {
            const int j = l - 4;
            float v[8];
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] = co[(1 + j * 2) * 8 + k];
            if (j == 0) v[0] = dcs2;
            idct1d<8>(v);
#pragma unroll
            for (int x = 0; x < 8; x++) tmp[16 + j * 8 + x] = v[x];
          }
          __syncwarp();
          if (l < 4) {
            float u[4];
#pragma unroll
            for (int j = 0; j < 4; j++) u[j] = tmp[j * 4 + l];
            idct1d<4>(u);
            if (JXLB_PX_OK) {
#pragma unroll
              for (int yy = 0; yy < 4; yy++) px[(afv_y * 4 + yy) * PP + (afv_x == 1 ? 0 : 4) + l] = u[yy];
            }
          }
          {
            float u[4];
#pragma unroll
            for (int j = 0; j < 4; j++) u[j] = tmp[16 + j * 8 + l];
            idct1d<4>(u);
            if (JXLB_PX_OK) {
#pragma unroll
              for (int yy = 0; yy < 4; yy++) px[((afv_y == 1 ? 0 : 4) + yy) * PP + l] = u[yy];
            }
          }
          break;
        }
      }
    }
    out.finish(c, l, active);
  }
#undef JXLB_PX_OK
}

// 8x8-class varblocks (DCT and the specials): 8 lanes per block, 4 blocks per warp.
// Phase A: lane l loads its column (DCT8x8) or row (the specials) of all three channels and dequantises
// them in registers (CfL needs Y next to X and B anyway).
// Phase B: the strategy's transform (block8_transform).
// vec: the coefficient planes are 16-byte aligned (rows of the specials as vector loads, see load_lane8).
template <bool I32>
__device__ __forceinline__ void block8_item(const FrameDev& P, int kind, uint4 entry, bool active,
                                            uint4 entry_next, bool next_active, bool vec, float* sm) {
  const int lane = threadIdx.x & 31;
  const int slot = lane >> 3, l = lane & 7;
  // Inactive slots (tail of a list) run the same instruction stream on scratch data so that
  // every __syncwarp() is reached by all 32 lanes; only their loads and stores are masked.
  float* scr = sm + slot * 264;   // 264 = 192 + 64 + 8: slot bases 8 banks apart
  VarblockCtx vb;
  float val[3][8];
  if (active) {
    vb = make_ctx(P, entry);
    const bool col = kind == 0;
    block8_dequant(P, kind, vb, l, col,
                   [&](int c, int* q) { load_lane8<I32>(P.coeff[c], vb.cbase, l, col, vec, q); }, val);
  } else {
    vb = VarblockCtx{};
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
      for (int e = 0; e < 8; e++) val[c][e] = 0.0f;
  }
  // Pull the NEXT item's coefficient lines (streamed from HBM exactly once) into L2 while this
  // item is being transformed: no registers are held, the next item's loads become L2 hits.
  if (next_active) {
    constexpr int kLines = I32 ? 2 : 1;  // a block-channel is 256 / 128 contiguous bytes
    if (l < 3 * kLines) {
      const int ch = l / kLines, half = l % kLines;
      const char* p = reinterpret_cast<const char*>(P.coeff[ch]) +
                      ((size_t)entry_next.y * 64u) * (I32 ? 4 : 2) + half * 128;
#if JXLB_PTX
      asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
      (void)p;
#endif
    }
  }
  Block8ToPlanes out;
  out.scratch = scr + 192;
  out.plane0 = P.xyb + (size_t)vb.aby * 8 * P.row_stride + vb.abx * 8;
  out.plane_stride = P.plane_stride;
  out.row_stride = P.row_stride;
  block8_transform(kind, active, val, l, scr, out);
}

constexpr int kSmallWarpsPerCta = 8;
constexpr int kSmallWarpFloats = 1120;  // >= 32*33 + 2*16 and >= 4*264

__device__ __forceinline__ int small_slots(int s) {
  const int w = max(covered_x(s), covered_y(s));
  return w == 1 ? 4 : (w == 2 ? 2 : 1);
}

// 8x8-class strategies (DCT, IDENTITY, DCT2X2, DCT4X4, DCT4X8, DCT8X4, AFV0-3).  Takes any element-aligned
// coefficient planes (device-resident planes of a caller need not be 16-byte aligned).
template <bool I32>
__global__ void __launch_bounds__(kSmallWarpsPerCta * 32, 4) idct8_kernel(const __grid_constant__ FrameDev P) {
  __shared__ __align__(16) float smem[kSmallWarpsPerCta * 1056];
  float* sm = smem + (threadIdx.x >> 5) * 1056;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  const bool vec = (((uintptr_t)P.coeff[0] | (uintptr_t)P.coeff[1] | (uintptr_t)P.coeff[2]) & 15u) == 0;
  const int order[10] = {0, 2, 12, 13, 1, 3, 14, 15, 16, 17};
  uint32_t base = 0;
#pragma unroll 1
  for (int oi = 0; oi < 10; oi++) {
    const int s = order[oi];
    const uint32_t count = P.counts[s];
    const uint32_t items = (count + 3) / 4;
    uint32_t it = (warp + nwarps - (base % nwarps)) % nwarps;
    const int slot = (threadIdx.x & 31) >> 3;
    const uint4* list = P.list + P.list_base[s];
    const uint4 zero = make_uint4(0, 0, 1, 0);
    bool act = it < items && it * 4 + slot < count;
    uint4 cur = act ? __ldg(list + it * 4 + slot) : zero;
    {
#pragma unroll 1
      for (; it < items; it += nwarps) {
        const uint32_t nx = (it + nwarps) * 4 + slot;  // the record of this warp's next item is fetched now
        const bool nact = (it + nwarps) < items && nx < count;
        const uint4 next = nact ? __ldg(list + nx) : zero;
        block8_item<I32>(P, s, cur, act, next, nact, vec, sm);
        cur = next;
        act = nact;
      }
    }
    base += items;
  }
}

// multi-block DCTs with sides <= 32 (DCT16X16 .. DCT16X32).
// ---------------------------------------------------------------------------
// idct8_tma_kernel: the same items as idct8_kernel, with the coefficients staged by the bulk-copy (TMA)
// unit.  idct8_kernel is latency bound (ncu: 8 long-scoreboard stall cycles per issue, 57 % of the HBM
// peak): a warp loads the 3 x 256 bytes of each of its four blocks with ordinary loads and waits for them.
// Here every warp owns two staging buffers of 4 blocks x 192 words in shared memory and an mbarrier each;
// while item i is transformed, the 12 block-channels of item i+1 (the warp's next item, possibly of the next
// strategy list) are already in flight as cp.async.bulk copies (global -> shared, complete_tx on the
// barrier), issued by 12 lanes as soon as buffer (i+1)&1 is free.  After dequantisation (all of a block's
// coefficients sit in registers) the staging words serve as the transform's scratch, like in the fused
// kernel, pixel scratch of the specials included.
// Nothing a warp waits for on its way through an item is fetched late: the work-list record is loaded three
// items ahead into shared memory (cp.async: no register is held while it is in flight), the block's three DC
// values two items ahead (with the copies, by three otherwise idle lanes, handed over by shuffle), the list
// sizes sit in shared memory.  2 CTAs x 16 warps per SM (64 registers without spills, 112 KB of shared memory
// per CTA) keep 32 warps and ~100 KB of coefficient reads in flight per SM.
// Needs 16-byte aligned coefficient planes (jxlgpu_set_device_coefficients may bring others: idct8_kernel).
// ---------------------------------------------------------------------------
constexpr int kTma8Warps = 16;
constexpr int kTma8BlockWords = 200;  // 3 channels x 64 int32 (int16: half used) + 8: the four blocks of a warp start 8 banks apart
constexpr int kTma8StageWords = 4 * kTma8BlockWords;
constexpr int kTma8WarpWords = 2 * kTma8StageWords + 4;        // 2 stages | 2 mbarriers
constexpr size_t kTma8SmemBytes = (size_t)kTma8Warps * kTma8WarpWords * 4;

template <bool I32>
__global__ void __launch_bounds__(kTma8Warps * 32, 2) idct8_tma_kernel(const __grid_constant__ FrameDev P) {
  extern __shared__ __align__(16) float fsm[];
  uint32_t* wsm = reinterpret_cast<uint32_t*>(fsm) + (threadIdx.x >> 5) * kTma8WarpWords;
  uint64_t* bars = reinterpret_cast<uint64_t*>(wsm + 2 * kTma8StageWords);
  const int lane = threadIdx.x & 31, slot = lane >> 3, l = lane & 7;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  constexpr uint32_t kChBytes = I32 ? 256 : 128;
  constexpr int kChWords = I32 ? 64 : 32;
  // the ten 8x8-class work lists as one index space: items [pre[i], pre[i+1]) belong to strategy skind[i],
  // whose list holds cnt[i] records; the ten strategies' dequant matrices (3 x 64 floats each) are copied to
  // shared memory once per CTA
  __shared__ uint32_t pre[11], cnt[10];
  __shared__ int skind[10];
  __shared__ __align__(16) float sdq[10 * 192];
  // per warp, the work-list records of its current item and the three after it (ring of 4 items x 4 slots)
  __shared__ __align__(16) uint4 srec[kTma8Warps * 16];
  uint4* recs = srec + (threadIdx.x >> 5) * 16;
  {
    const int order[10] = {0, 2, 12, 13, 1, 3, 14, 15, 16, 17};
    if (threadIdx.x == 0) {
      uint32_t acc = 0;
      for (int i = 0; i < 10; i++) {
        pre[i] = acc;
        skind[i] = order[i];
        cnt[i] = P.counts[order[i]];
        acc += (cnt[i] + 3) / 4;
      }
      pre[10] = acc;
    }
    for (int e = threadIdx.x; e < 10 * 192; e += blockDim.x) {
      const int i = e / 192, c = (e % 192) / 64, k = e % 64;
      int s_ = 0;
#pragma unroll
      for (int q = 0; q < 10; q++) s_ = (q == i) ? order[q] : s_;
      sdq[e] = __ldg(P.dq + P.dq_off[3 * s_ + c] + k);
    }
  }
  if (lane == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
  }
  fence_async_smem();
  __syncthreads();
  const uint32_t total = pre[10];

  // item v (warp-uniform): its list index (-1 past the end; recomputed where needed rather than held in
  // registers -- the lists are in order and most items belong to the first) and whether the slot has a block
  auto list_of = [&](uint32_t v) {
    if (v >= total) return -1;
    int oi = 0;
    while (v >= pre[oi + 1]) oi++;
    return oi;
  };
  auto is_act = [&](uint32_t v, int oi) {
    if (oi < 0) return false;
    return (v - pre[oi]) * 4 + slot < cnt[oi];
  };
  // lane 6 of each slot copies the slot's record of item v into ring position `pos` (cp.async, one commit
  // group per call; a zero record for the inactive slots at a list's tail and past the end), three items
  // before the item is transformed
  const uint4 zero = make_uint4(0, 0, 1, 0);
  auto fetch_rec = [&](uint32_t v, int pos) {
    const int oi = list_of(v);
    if (l == 6) {
      if (is_act(v, oi)) async_copy16(recs + pos * 4 + slot, P.list + P.list_base[skind[oi]] + (v - pre[oi]) * 4 + slot);
      else recs[pos * 4 + slot] = zero;
    }
    async_commit();
  };
  // (a record's third word is the raw quantiser: 0 never occurs, so zero.z == 1 with y == 0 marks "inactive"
  //  only through the explicit flag below)
  // Lanes 0..2 of a slot copy channel l of its block; lanes 3..5 load DC value l - 3 of the block into `dc`.
  auto issue = [&](int st, int pos, bool act, float& dc) {
    const uint32_t nact = __popc(__ballot_sync(0xffffffffu, act && l == 0));
    if (nact == 0) return;
    if (lane == 0) mbar_arrive_expect_tx(&bars[st], nact * 3 * kChBytes);
    __syncwarp();
    const uint4 rec = recs[pos * 4 + slot];
    if (act && l < 3) {
      char* dst = reinterpret_cast<char*>(wsm + st * kTma8StageWords + slot * kTma8BlockWords) + l * kChBytes;
      const void* plane = l == 0 ? P.coeff[0] : (l == 1 ? P.coeff[1] : P.coeff[2]);
      const char* src = reinterpret_cast<const char*>(plane) + (size_t)rec.y * 64u * (I32 ? 4 : 2);
      bulk_g2s(dst, src, kChBytes, &bars[st]);
    }
    if (act && l >= 3 && l < 6)
      dc = __ldg(P.dc + (size_t)(l - 3) * P.yb * P.xb + (size_t)(rec.x >> 16) * P.xb + (rec.x & 0xffffu));
  };

  uint32_t v = warp;
  float dc_cur = 0.0f, dc_next = 0.0f;  // lanes 3..5: DC value l - 3 of this item's / the next item's block
  fetch_rec(v, 0);
  fetch_rec(v + nwarps, 1);
  fetch_rec(v + 2 * nwarps, 2);
  async_wait<0>();
  __syncwarp();
  issue(0, 0, is_act(v, list_of(v)), dc_cur);
  issue(1, 1, is_act(v + nwarps, list_of(v + nwarps)), dc_next);
  // ring position of item v: its staging buffer is st = pos & 1, whose completion of this item has
  // parity (pos >> 1) & 1 (each buffer takes every other item)
  uint32_t pos = 0;
#pragma unroll 1
  for (; v < total; v += nwarps, pos = (pos + 1) & 3u) {
    const int st = pos & 1;
    // the record of the item three ahead starts its trip now; it is used (for the copies) next iteration
    fetch_rec(v + 3 * nwarps, (pos + 3) & 3u);
    const int oi_cur = list_of(v);
    const bool act_cur = is_act(v, oi_cur);
    const int kind = skind[oi_cur];
    float dc[3];
#pragma unroll
    for (int c = 0; c < 3; c++) dc[c] = __shfl_sync(0xffffffffu, dc_cur, (lane & ~7) + 3 + c);
    mbar_wait(&bars[st], (pos >> 1) & 1u);
    uint32_t* stg = wsm + st * kTma8StageWords + slot * kTma8BlockWords;
    float* scr = reinterpret_cast<float*>(stg);
    VarblockCtx vb;
    float val[3][8];
    if (act_cur) {
      vb = make_ctx(P, recs[pos * 4 + slot]);
      const bool col = kind == 0;
      const float* dqm = sdq + oi_cur * 192;
      block8_dequant_m<true>(P, dqm, dqm + 64, dqm + 128, vb, l, col,
                             [&](int c, int* q) { load_lane8_smem<I32>(stg + c * kChWords, l, col, q); }, val);
      if (l == 0) {
#pragma unroll
        for (int c = 0; c < 3; c++) val[c][0] = dc[c];
      }
    } else {
      vb = VarblockCtx{};
#pragma unroll
      for (int c = 0; c < 3; c++)
#pragma unroll
        for (int e = 0; e < 8; e++) val[c][e] = 0.0f;
    }
    __syncwarp();  // every lane holds its coefficients: the staging words become the transform's scratch
    Block8ToPlanes out;
    out.scratch = scr + 128;
    out.plane0 = P.xyb + (size_t)vb.aby * 8 * P.row_stride + vb.abx * 8;
    out.plane_stride = P.plane_stride;
    out.row_stride = P.row_stride;
    block8_transform(kind, act_cur, val, l, scr, out);
    // buffer `st` is free: the item after next goes there (its record, fetched last iteration, has landed)
    fence_async_smem();
    async_wait<1>();
    __syncwarp();
    dc_cur = dc_next;
    issue(st, (pos + 2) & 3u, is_act(v + 2 * nwarps, list_of(v + 2 * nwarps)), dc_next);
  }
}

template <bool I32>
__global__ void __launch_bounds__(kSmallWarpsPerCta * 32) idct_mid_kernel(const __grid_constant__ FrameDev P) {
  __shared__ __align__(16) float smem[kSmallWarpsPerCta * kSmallWarpFloats];
  float* sm = smem + (threadIdx.x >> 5) * kSmallWarpFloats;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  // warp items are numbered class by class; larger transforms first for balance
  const int order[8] = {5, 10, 11, 8, 9, 4, 6, 7};
  uint32_t base = 0;
#pragma unroll 1
  for (int oi = 0; oi < 8; oi++) {
    const int s = order[oi];
    const uint32_t count = P.counts[s];
    const uint32_t slots = small_slots(s);
    const uint32_t items = (count + slots - 1) / slots;
    uint32_t it = (warp + nwarps - (base % nwarps)) % nwarps;
#pragma unroll 1
    for (; it < items; it += nwarps) {
      const uint32_t e0 = it * slots;
      switch (s) {
        case 4: small_dct_item<16, 16, I32>(P, s, e0, count, sm); break;
        case 5: small_dct_item<32, 32, I32>(P, s, e0, count, sm); break;
        case 6: small_dct_item<16, 8, I32>(P, s, e0, count, sm); break;
        case 7: small_dct_item<8, 16, I32>(P, s, e0, count, sm); break;
        case 8: small_dct_item<32, 8, I32>(P, s, e0, count, sm); break;
        case 9: small_dct_item<8, 32, I32>(P, s, e0, count, sm); break;
        case 10: small_dct_item<32, 16, I32>(P, s, e0, count, sm); break;
        default: small_dct_item<16, 32, I32>(P, s, e0, count, sm); break;
      }
    }
    base += items;
  }
}

// ---------------------------------------------------------------------------
// large IDCT: one CTA (256 threads) per varblock with a 64/128/256 side.
// Pass 1 writes the horizontally transformed rows into the varblock's own region of
// the output plane; pass 2 transforms the columns in place.
// ---------------------------------------------------------------------------
// Warp-cooperative N-point IDCTs (N = 128, 256) on TOT / N vectors stored back to back in shared memory
// (a segment of the recursion never straddles two vectors, so the batch is just a longer index range):
// recursion levels down to 32-point leaves done by all lanes, leaves in registers, one leaf per lane --
// with TOT = 1024 every lane has a leaf.
template <int N, int TOT>
__device__ __forceinline__ void idct1d_warp(float* v /*TOT*/, float* w /*TOT scratch*/) {
  const int lane = threadIdx.x & 31;
  // top-down: even/odd split + BTranspose of the odd half, sizes N, N/2, ..., 64
  float* src = v;
  float* dst = w;
#pragma unroll
  for (int n = N; n > 32; n >>= 1) {
    const int h = n >> 1;
    for (int i = lane; i < TOT; i += 32) {
      const int seg = i / n, r = i % n;  // element r of segment seg
      const float* s = src + seg * n;
      float val;
      if (r < h) {
        val = s[2 * r];
      } else {
        const int q = r - h;
        val = (q == 0) ? s[1] * kSqrt2 : (s[2 * q + 1] + s[2 * q - 1]);
      }
      dst[i] = val;
    }
    __syncwarp();
    float* t = src; src = dst; dst = t;
  }
  // leaves: TOT/32 independent 32-point IDCTs
  if (lane < TOT / 32) {
    float r[32];
#pragma unroll
    for (int i = 0; i < 32; i++) r[i] = src[lane * 32 + i];
    idct1d<32>(r);
#pragma unroll
    for (int i = 0; i < 32; i++) src[lane * 32 + i] = r[i];
  }
  __syncwarp();
  // bottom-up: MultiplyAndAdd, sizes 64, ..., N
#pragma unroll
  for (int n = 64; n <= N; n <<= 1) {
    const int h = n >> 1;
    for (int i = lane; i < TOT / 2; i += 32) {
      const int seg = i / h, r = i % h;
      const float* s = src + seg * n;
      const float wv = JXT_WC[h - 2 + r];
      const float e = s[r], o = s[h + r];
      dst[seg * n + r] = fmaf(wv, o, e);
      dst[seg * n + n - 1 - r] = fmaf(-wv, o, e);
    }
    __syncwarp();
    float* t = src; src = dst; dst = t;
  }
  if (src != v) {
    for (int i = lane; i < TOT; i += 32) v[i] = src[i];
    __syncwarp();
  }
}

// Work items of the two passes.  A 256x256 varblock is 196 K coefficients: one CTA per varblock (round 1)
// left the handful of largest varblocks of a frame running alone for milliseconds, so each pass is cut into
// slabs -- pass 0: rows of one channel, pass 1: columns of one channel -- that spread over the grid, and the
// two passes are two launches (the only dependency between them is per varblock).
constexpr int kLargeWarps = 8;
template <int R, int C>
__host__ __device__ constexpr int large_rows_per_item() { return C <= 64 ? 256 : kLargeWarps * (1024 / C); }
template <int R, int C>
__host__ __device__ constexpr int large_slabs(int pass) {
  return pass == 0 ? (3 * R + large_rows_per_item<R, C>() - 1) / large_rows_per_item<R, C>()
                   : (R <= 64 ? (3 * C + 255) / 256 : 3 * C / 32);
}
// shared memory (floats): llf 1024 | llf_tmp 1024 | per-warp transform buffers 8 x 2048 | (pass 1) a
// [R][33] tile of 32 columns, aliasing the LLF area and growing past the buffers
constexpr int kLargeCoopOff = 2048;
constexpr int kLargeTileOff = kLargeCoopOff + kLargeWarps * 2048;
constexpr int kLargeSmemFloats = kLargeTileOff + 256 * 33;

template <int R, int C, bool I32, int PASS>
__device__ __forceinline__ void large_item(const FrameDev& P, int kind, uint4 entry, int slab, float* sm) {
  constexpr int CY = R / 8, CX = C / 8;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  float* llf = sm;                   // <= 1024 floats
  float* llf_tmp = sm + 1024;        // CY*CX
  float* coop = sm + kLargeCoopOff;  // 8 warps * 2 * 1024
  const VarblockCtx vb = make_ctx(P, entry);
  if constexpr (PASS == 0) {
    // ---- pass 0: rows (c, j): IDCT over horizontal frequency, into the varblock's region of the planes ----
    if constexpr (C <= 64) {
      for (int c = 0; c < 3; c++)  // (tiny: at most 16 x 8 values per channel)
        llf_from_dc<CY, CX>(P.dc + (size_t)c * P.yb * P.xb + (size_t)vb.aby * P.xb + vb.abx, P.xb, tid,
                            llf_tmp, llf + c * CY * CX, BlockSync());
      const int r = slab * 256 + tid;
      if (r < 3 * R) {
        const int c = r / R, j = r % R;
        float v[C];
#pragma unroll
        for (int k = 0; k < C; k++) {
          const uint32_t i = (R >= C) ? (uint32_t)(k * R + j) : (uint32_t)(j * C + k);
          v[k] = dequant<I32>(P, vb, kind, c, i);
        }
        if (j < CY) {
#pragma unroll
          for (int k = 0; k < CX; k++) v[k] = llf[c * CY * CX + j * CX + k];
        }
        idct1d<C>(v);
        float* out = P.xyb + (size_t)c * P.plane_stride + ((size_t)vb.aby * 8 + j) * P.row_stride + vb.abx * 8;
#pragma unroll
        for (int x = 0; x < C; x += 4)
          *reinterpret_cast<float4*>(out + x) = make_float4(v[x], v[x + 1], v[x + 2], v[x + 3]);
      }
    } else {
      constexpr int NB = 1024 / C;                 // rows per warp
      constexpr int RPI = kLargeWarps * NB;        // rows per item, all of one channel (R % RPI == 0)
      static_assert(R % RPI == 0, "a slab stays inside one channel");
      const int c = (slab * RPI) / R, j0 = (slab * RPI) % R;
      if (j0 == 0)  // the slab holds the rows with the lowest vertical frequencies
        llf_from_dc<CY, CX>(P.dc + (size_t)c * P.yb * P.xb + (size_t)vb.aby * P.xb + vb.abx, P.xb, tid,
                            llf_tmp, llf, BlockSync());
      float* buf = coop + warp * 2048;
      const int jw = j0 + warp * NB;
      for (int e = lane; e < NB * C; e += 32) {
        const int b = e / C, k = e % C, j = jw + b;
        const uint32_t i = (R >= C) ? (uint32_t)(k * R + j) : (uint32_t)(j * C + k);
        float val = dequant<I32>(P, vb, kind, c, i);
        if (j < CY && k < CX) val = llf[j * CX + k];
        buf[e] = val;
      }
      __syncwarp();
      idct1d_warp<C, 1024>(buf, buf + 1024);
      for (int b = 0; b < NB; b++) {
        float* out = P.xyb + (size_t)c * P.plane_stride + ((size_t)vb.aby * 8 + jw + b) * P.row_stride + vb.abx * 8;
        for (int x = lane; x < C; x += 32) out[x] = buf[b * C + x];
      }
      __syncwarp();
    }
  } else {
    // ---- pass 1: columns (c, x): IDCT over vertical frequency, in place ----
    if constexpr (R <= 64) {
      const int r = slab * 256 + tid;
      if (r < 3 * C) {
        const int c = r / C, x = r % C;
        float* col = P.xyb + (size_t)c * P.plane_stride + (size_t)vb.aby * 8 * P.row_stride + vb.abx * 8 + x;
        float u[R];
#pragma unroll
        for (int j = 0; j < R; j++) u[j] = col[(size_t)j * P.row_stride];
        idct1d<R>(u);
#pragma unroll
        for (int y = 0; y < R; y++) col[(size_t)y * P.row_stride] = u[y];
      }
    } else {
      // 32 columns of one channel: the [R][32] tile travels between the plane and shared memory in
      // full 128-byte rows; each warp transforms 4 of its columns at a time
      constexpr int XS = C / 32;  // column slabs per channel
      const int c = slab / XS, x0 = (slab % XS) * 32;
      float* tile = sm + kLargeTileOff;  // [R][33]
      float* base = P.xyb + (size_t)c * P.plane_stride + (size_t)vb.aby * 8 * P.row_stride + vb.abx * 8 + x0;
      for (int j = warp; j < R; j += kLargeWarps) tile[j * 33 + lane] = base[(size_t)j * P.row_stride + lane];
      __syncthreads();
      float* buf = coop + warp * 2048;
      for (int e = lane; e < 4 * R; e += 32) buf[e] = tile[(e % R) * 33 + 4 * warp + e / R];
      __syncwarp();
      idct1d_warp<R, 4 * R>(buf, buf + 1024);
      for (int e = lane; e < 4 * R; e += 32) tile[(e % R) * 33 + 4 * warp + e / R] = buf[e];
      __syncthreads();
      for (int j = warp; j < R; j += kLargeWarps) base[(size_t)j * P.row_stride + lane] = tile[j * 33 + lane];
    }
  }
  __syncthreads();
}

template <bool I32, int PASS>
__global__ void __launch_bounds__(kLargeWarps * 32) idct_large_kernel(const __grid_constant__ FrameDev P) {
  extern __shared__ __align__(16) float fsm[];
  float* sm = fsm;
  uint32_t base = 0;
#pragma unroll 1
  for (int s = kNumStrategies - 1; s >= kFirstLarge; s--) {
    int slabs;
    switch (s) {
      case 18: slabs = large_slabs<64, 64>(PASS); break;
      case 19: slabs = large_slabs<64, 32>(PASS); break;
      case 20: slabs = large_slabs<32, 64>(PASS); break;
      case 21: slabs = large_slabs<128, 128>(PASS); break;
      case 22: slabs = large_slabs<128, 64>(PASS); break;
      case 23: slabs = large_slabs<64, 128>(PASS); break;
      case 24: slabs = large_slabs<256, 256>(PASS); break;
      case 25: slabs = large_slabs<256, 128>(PASS); break;
      default: slabs = large_slabs<128, 256>(PASS); break;
    }
    const uint32_t count = P.counts[s] * (uint32_t)slabs;
    uint32_t it = (blockIdx.x + gridDim.x - (base % gridDim.x)) % gridDim.x;
#pragma unroll 1
    for (; it < count; it += gridDim.x) {
      const uint4 entry = __ldg(P.list + P.list_base[s] + it / (uint32_t)slabs);
      const int slab = (int)(it % (uint32_t)slabs);
      switch (s) {
        case 18: large_item<64, 64, I32, PASS>(P, s, entry, slab, sm); break;
        case 19: large_item<64, 32, I32, PASS>(P, s, entry, slab, sm); break;
        case 20: large_item<32, 64, I32, PASS>(P, s, entry, slab, sm); break;
        case 21: large_item<128, 128, I32, PASS>(P, s, entry, slab, sm); break;
        case 22: large_item<128, 64, I32, PASS>(P, s, entry, slab, sm); break;
        case 23: large_item<64, 128, I32, PASS>(P, s, entry, slab, sm); break;
        case 24: large_item<256, 256, I32, PASS>(P, s, entry, slab, sm); break;
        case 25: large_item<256, 128, I32, PASS>(P, s, entry, slab, sm); break;
        default: large_item<128, 256, I32, PASS>(P, s, entry, slab, sm); break;
      }
    }
    base += count;
  }
}

// ---------------------------------------------------------------------------
// DC stage (optional, SURVEY.md §8f rank 2): dequantise the quantised DC image and smooth it on the
// device instead of uploading finished float planes.  One thread per 8x8 block; the arithmetic lives
// in jxl_dc_stage.h (shared with a host-side test).  Tiny: 0.5 M blocks at 8K.
// ---------------------------------------------------------------------------
#ifndef JXLB_STRIP_TU
__global__ void __launch_bounds__(256) dc_dequant_kernel(const __grid_constant__ DcStage S) {
  const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x < S.xb && y < S.yb) dc_dequant_px(S, x, y);
}
__global__ void __launch_bounds__(256) dc_smooth_kernel(const __grid_constant__ DcStage S, int smoothing) {
  const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x < S.xb && y < S.yb) dc_smooth_px(S, x, y, smoothing != 0);
}
#endif  // JXLB_STRIP_TU

// ---------------------------------------------------------------------------
// Sparse coefficient hand-off (jxlgpu_submit_groups_sparse): scatter the non-zero entries of up to
// kMaxSparseSegs (group, channel) lists into the zero-filled dense planes.  HBM-bound: 4 bytes read
// and one 2/4-byte store per non-zero; the stores of one varblock fall into few 32-byte sectors
// because the low frequencies, where the non-zeros are, sit together in the natural order.
// ---------------------------------------------------------------------------
struct SparseSeg {
  uint32_t src_off;  // first word of the list inside the staging buffer
  uint32_t n;        // entries
  uint32_t dst_off;  // first element of the (group, channel) plane inside the dense buffer
  uint32_t wide;     // 0: (pos << 16) | u16 value words; 1: {pos, value} word pairs
};
constexpr int kMaxSparseSegs = 192;
struct SparseBatch {
  SparseSeg seg[kMaxSparseSegs];
};

#ifndef JXLB_STRIP_TU
// ---------------------------------------------------------------------------
// Multi-GPU gather, SM variant (JXLGPU_GATHER=sm): one launch copies a finished row chunk of this rank's band to
// the same offset of every peer's frame buffer (peer-mapped symmetric memory) with 16-byte loads and stores;
// a warp writes 512 contiguous bytes per peer and instruction, CTAs start at different peers.
// ---------------------------------------------------------------------------
struct PeerDst {
  char* p[8];
  uint32_t n;
};
__global__ void __launch_bounds__(256) peer_copy_kernel(const char* __restrict__ src, const __grid_constant__ PeerDst dst,
                                                        size_t bytes) {
  const size_t n16 = bytes / 16;
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  const uint32_t first = blockIdx.x % (dst.n ? dst.n : 1);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) {
    const uint4 v = s4[i];
#pragma unroll 1
    for (uint32_t k = 0; k < dst.n; k++) {
      uint32_t q = first + k;
      if (q >= dst.n) q -= dst.n;
      reinterpret_cast<uint4*>(dst.p[q])[i] = v;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (bytes & 15)) {  // tail
    const size_t i = n16 * 16 + threadIdx.x;
    for (uint32_t q = 0; q < dst.n; q++) dst.p[q][i] = src[i];
  }
}

template <bool I32>
__global__ void __launch_bounds__(256) sparse_expand_kernel(const __grid_constant__ SparseBatch B,
                                                            const uint32_t* __restrict__ staging,
                                                            void* __restrict__ coeff) {
  const SparseSeg sg = B.seg[blockIdx.y];
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < sg.n; i += gridDim.x * blockDim.x) {
    uint32_t pos;
    int32_t val;
    if (sg.wide) {
      const uint2 w = *reinterpret_cast<const uint2*>(staging + sg.src_off + 2 * (size_t)i);
      pos = w.x;
      val = (int32_t)w.y;
    } else {
      const uint32_t w = staging[sg.src_off + i];
      pos = w >> 16;
      val = (int32_t)(int16_t)(w & 0xffffu);
    }
    if (pos < 65536u) {
      if constexpr (I32) reinterpret_cast<int32_t*>(coeff)[(size_t)sg.dst_off + pos] = val;
      else reinterpret_cast<int16_t*>(coeff)[(size_t)sg.dst_off + pos] = (int16_t)val;
    }
  }
}
#endif  // JXLB_STRIP_TU

// ---------------------------------------------------------------------------
// fused filter kernel: [Gaborish] -> [EPF0] -> [EPF1] -> [EPF2] -> [XYB->linear RGB]
// One CTA per TW x TH output tile; every enabled stage is evaluated on a shrinking
// halo inside two shared-memory ping-pong tiles.  Positions outside the image are
// never computed: reads are redirected to their mirror image inside the tile
// (Mirror(), lib/jxl/image_ops.h:184-196 -- every stage's input is mirrored about the
// true image size, simple_render_pipeline.cc:129-164).
// ---------------------------------------------------------------------------
// Fused all-gather (multi-GPU).  A filter CTA first writes its strip segment into this rank's slot
// of the LOCAL frame buffer, then -- while other CTAs are still filtering -- replays that region
// (hot in L2) to every peer with wide, fully coalesced stores: one multimem.st.v2 per 8 bytes through
// the NVSwitch multicast mapping (the switch replicates it to all GPUs), or plain peer stores over
// NVLink P2P.  The transfer therefore overlaps the math segment by segment and no separate
// collective kernel runs.
__device__ __forceinline__ void mc_store2(float* p, float2 v) {
#if JXLB_PTX
  asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v.x), "f"(v.y) : "memory");
#else
  reinterpret_cast<float2*>(p)[0] = v;  // (no switch to replicate it: a plain store)
#endif
}
__device__ __forceinline__ void mc_store1(float* p, float v) {
#if JXLB_PTX
  asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
#else
  *p = v;
#endif
}

// replicate `n` bytes starting at byte offset `off` of the local buffer `src` (all threads of the
// CTA): bytes up to the first 8-byte boundary, an 8-byte vector body, the remaining bytes.  The
// multicast mapping takes 4-byte granules only (f32 layouts; the host rejects it otherwise).
__device__ __forceinline__ void replicate_span(const FrameDev& P, const char* src, size_t off, int n) {
  const int tid = threadIdx.x, nt = blockDim.x;
  int head = (int)((8 - (off & 7)) & 7);
  if (head > n) head = n;
  const int nv = (n - head) >> 3;
  const int tail = n - head - 8 * nv;
  if (P.mc) {
    if (tid == 0) {
      if (head) mc_store1(reinterpret_cast<float*>(P.mc + off), *reinterpret_cast<const float*>(src + off));
      if (tail) {
        const size_t o = off + head + 8 * (size_t)nv;
        mc_store1(reinterpret_cast<float*>(P.mc + o), *reinterpret_cast<const float*>(src + o));
      }
    }
  } else if (tid < head + tail) {
    const size_t o = tid < head ? off + tid : off + head + 8 * (size_t)nv + (tid - head);
    const char v = src[o];
    for (uint32_t i = 0; i < P.nrep; i++) P.rep[i][o] = v;
  }
  const float2* s2 = reinterpret_cast<const float2*>(src + off + head);
  for (int i = tid; i < nv; i += nt) {
    const float2 v = s2[i];
    const size_t o = off + head + 8 * (size_t)i;
    if (P.mc) {
      mc_store2(reinterpret_cast<float*>(P.mc + o), v);
    } else {
#pragma unroll 1
      for (uint32_t k = 0; k < P.nrep; k++) *reinterpret_cast<float2*>(P.rep[k] + o) = v;
    }
  }
}

// bytes per pixel of the interleaved JXLGPU_OUT_* layouts (bytes per sample for the planar one)
__host__ __device__ constexpr int out_pixel_bytes(uint32_t fmt) {
  return fmt == 0 ? 12 : fmt == 1 ? 4 : fmt == 2 ? 3 : fmt == 3 ? 4 : 6;
}

// TF_SRGB::EncodedFromDisplay (cms/transfer_functions-inl.h:244-267): what FromLinearStage<OpRgb>
// applies with JXL_HIGH_PRECISION (stage_from_linear.cc:42-53).  IEEE sqrt and division, Horner
// with FMAs (rational_polynomial-inl.h:59-97) -- bit-exact against the CPU.
// kYCbCrStage (lib/jxl/render_pipeline/stage_ycbcr.cc:33-71): full-range BT.601; a = Cb, b = Y, c3 = Cr in, R, G, B out
__device__ __forceinline__ void ycbcr_px(float& a, float& b, float& c3) {
  const float c128 = 128.0f / 255, crcr = 1.402f, cgcb = -0.114f * 1.772f / 0.587f, cgcr = -0.299f * 1.402f / 0.587f,
              cbcb = 1.772f;
  const float yv = b + c128, cb = a, cr = c3;
  a = fmaf(crcr, cr, yv);
  b = fmaf(cgcr, cr, fmaf(cgcb, cb, yv));
  c3 = fmaf(cbcb, cb, yv);
}

__device__ __forceinline__ float srgb_from_linear(float v) {
  const float x = fabsf(v);
  const float s = __fsqrt_rn(x);
  float yp = 7.352629620e-01f, yq = 2.424867759e-02f;
  yp = fmaf(yp, s, 1.474205315e+00f); yq = fmaf(yq, s, 9.258482155e-01f);
  yp = fmaf(yp, s, 3.903842876e-01f); yq = fmaf(yq, s, 1.340816930e+00f);
  yp = fmaf(yp, s, 5.287254571e-03f); yq = fmaf(yq, s, 3.036675394e-01f);
  yp = fmaf(yp, s, -5.135152395e-04f); yq = fmaf(yq, s, 1.004519624e-02f);
  const float poly = __fdiv_rn(yp, yq);
  const float mag = x > 0.0031308f ? poly : x * 12.92f;
  return copysignf(fabsf(mag), v);
}

// MakeUnsigned (stage_write.cc:455-479): scale, 8-bit ordered dither, clamp (NaN -> 0 as maxps
// does), round half to even.
template <int BITS>
__device__ __forceinline__ uint32_t make_unsigned(float v, int x, int y, int c) {
  constexpr float mul = (float)((1u << BITS) - 1u);
  v = v * mul;
  if constexpr (BITS == 8) v = v + __ldg(&JXT_DITHER[(y + 13 * c) & 31][(x + 23 * c) & 31]);
  float t = v > 0.0f ? v : 0.0f;
  t = t < mul ? t : mul;
  return (uint32_t)__float2int_rn(t);
}

// Last two stages of the pipeline for one pixel: optional sRGB transfer function and the
// WriteToOutputStage conversion + interleave (stage_write.cc:455-640).  `yo` = row inside `out`.
// OUTK 0: the instantiation for linear interleaved f32 (no run-time format dispatch in the loop);
// OUTK 1: every other transfer function / layout, selected at run time.
template <int OUTK>
__device__ __forceinline__ void store_px(const FrameDev& P, char* __restrict__ out, size_t out_row_bytes,
                                         int yo, int x, int band_h, float a, float b, float c3) {
  if constexpr (OUTK == 0) {
    float* o = reinterpret_cast<float*>(out + (size_t)yo * out_row_bytes) + (size_t)x * 3;
    o[0] = a; o[1] = b; o[2] = c3;
    return;
  }
  if constexpr (OUTK == 2) {  // EXPERIMENT: sRGB transfer function + dithered 8-bit RGB, no run-time dispatch
    const int y = yo + (int)P.out_y0;
    uint8_t* o = reinterpret_cast<uint8_t*>(out + (size_t)yo * out_row_bytes) + (size_t)x * 3;
    o[0] = (uint8_t)make_unsigned<8>(srgb_from_linear(a), x, y, 0);
    o[1] = (uint8_t)make_unsigned<8>(srgb_from_linear(b), x, y, 1);
    o[2] = (uint8_t)make_unsigned<8>(srgb_from_linear(c3), x, y, 2);
    return;
  }
  if (P.stage_mask & 32u) {
    a = srgb_from_linear(a);
    b = srgb_from_linear(b);
    c3 = srgb_from_linear(c3);
  }
  char* row = out + (size_t)yo * out_row_bytes;
  const int y = yo + (int)P.out_y0;
  switch (P.out_format) {
    case 0: {
      float* o = reinterpret_cast<float*>(row) + (size_t)x * 3;
      o[0] = a; o[1] = b; o[2] = c3;
    } break;
    case 1: {
      const size_t plane = (size_t)band_h * out_row_bytes;
      reinterpret_cast<float*>(row)[x] = a;
      reinterpret_cast<float*>(row + plane)[x] = b;
      reinterpret_cast<float*>(row + 2 * plane)[x] = c3;
    } break;
    case 2: {
      uint8_t* o = reinterpret_cast<uint8_t*>(row) + (size_t)x * 3;
      o[0] = (uint8_t)make_unsigned<8>(a, x, y, 0);
      o[1] = (uint8_t)make_unsigned<8>(b, x, y, 1);
      o[2] = (uint8_t)make_unsigned<8>(c3, x, y, 2);
    } break;
    case 3: {  // opaque alpha: MakeUnsigned(1.0) = 255 for every dither value
      const uint32_t w = make_unsigned<8>(a, x, y, 0) | (make_unsigned<8>(b, x, y, 1) << 8) |
                         (make_unsigned<8>(c3, x, y, 2) << 16) | 0xff000000u;
      reinterpret_cast<uint32_t*>(row)[x] = w;
    } break;
    case 4: {
      uint16_t* o = reinterpret_cast<uint16_t*>(row) + (size_t)x * 3;
      o[0] = (uint16_t)make_unsigned<16>(a, x, y, 0);
      o[1] = (uint16_t)make_unsigned<16>(b, x, y, 1);
      o[2] = (uint16_t)make_unsigned<16>(c3, x, y, 2);
    } break;
    default: {  // binary16, round to nearest even (stage_write.cc:590-640)
      __half* o = reinterpret_cast<__half*>(row) + (size_t)x * 3;
      o[0] = __float2half_rn(a);
      o[1] = __float2half_rn(b);
      o[2] = __float2half_rn(c3);
    } break;
  }
}

constexpr int kTW = 64, kTH = 32, kMaxHalo = 7;
constexpr int kSW = kTW + 2 * kMaxHalo;       // 78
constexpr int kSH = kTH + 2 * kMaxHalo;       // 46
constexpr int kSP = kSW + 1;                  // row pitch 79 (odd)
constexpr int kTilePlane = kSH * kSP;
constexpr int kFilterSmemFloats = 2 * 3 * kTilePlane;
constexpr int kFilterThreads = 256;

__device__ __forceinline__ int mirror_i(int x, int size) {
  while (x < 0 || x >= size) x = (x < 0) ? (-x - 1) : (2 * size - 1 - x);
  return x;
}

struct TileGeom {
  int x0, y0;      // image coordinate of tile-buffer position (0,0)
  int W, H;        // image size
  bool edge;       // tile buffer reaches outside the image
  // tile-buffer offset of image pixel (y, x) neighbour, with mirroring when needed
  __device__ __forceinline__ int at(int ty, int tx) const {
    if (edge) {
      ty = mirror_i(y0 + ty, H) - y0;
      tx = mirror_i(x0 + tx, W) - x0;
    }
    return ty * kSP + tx;
  }
};

__device__ __forceinline__ float epf_weight(float sad, float inv_sigma) {
  const float v = fmaf(sad, inv_sigma, 1.0f);
  return v < 0.0f ? 0.0f : v;
}

#ifndef JXLB_STRIP_TU
// What PreparePipeline puts behind the filters / the upsampling (dec_cache.cc:232-330), for one output pixel:
// [ConvolveNoise + AddNoise] -> XYB -> linear RGB [-> sRGB] -> output packing.
__device__ __forceinline__ float noise_strength(const FrameDev& P, float x) {  // StrengthEvalLut, stage_noise.cc:72-139
  float scaled = x * 6.0f;
  scaled = scaled > 0.0f ? scaled : 0.0f;
  float fl = floorf(scaled);
  float frac = scaled - fl;
  if (scaled >= 7.0f) {
    fl = 6.0f;
    frac = 1.0f;
  }
  const int i = (int)fl;
  float v = fmaf(P.noise_lut[i + 1] - P.noise_lut[i], frac, P.noise_lut[i]);
  v = v < 1.0f ? v : 1.0f;
  return v < 0.0f ? 0.0f : v;
}
__device__ __forceinline__ void finish_px(const FrameDev& P, char* __restrict__ out, size_t out_row_stride, int X, int Y,
                                          float a, float b, float c3) {
  if (P.noise) {
    const int OW = (int)P.out_w, OH = (int)P.out_hh;
    // (the planes hold the CONVOLVED noise: noise_conv_kernel ran once per frame, behind the generator)
    float rnd[3];
#pragma unroll
    for (int c = 0; c < 3; c++) rnd[c] = __ldg(P.noise_planes + ((size_t)c * OH + Y) * OW + X) * 0.22f;
    // AddNoiseStage (stage_noise.cc:140-251)
    const float in_g = b - a, in_r = b + a;
    const float sg = noise_strength(P, in_g * 0.5f), sr = noise_strength(P, in_r * 0.5f);
    const float red = sr * fmaf(0.0078125f, rnd[0], 0.9921875f * rnd[2]);
    const float green = sg * fmaf(0.0078125f, rnd[1], 0.9921875f * rnd[2]);
    const float sum = red + green;
    a = fmaf(P.cfl_base_x, sum, red - green) + a;
    b = b + sum;
    c3 = fmaf(P.cfl_base_b, sum, c3);
  }
  if ((P.stage_mask & 16u) && P.ycbcr) {
    ycbcr_px(a, b, c3);
  } else if (P.stage_mask & 16u) {  // XYB -> linear RGB (dec_xyb-inl.h:38-86)
    float gr = b + a, gg = b - a, gb = c3;
    gr = gr - P.opsin_cbrt[0];
    gg = gg - P.opsin_cbrt[1];
    gb = gb - P.opsin_cbrt[2];
    const float r2 = gr * gr, g2 = gg * gg, b2 = gb * gb;
    const float mr = fmaf(r2, gr, P.opsin_bias[0]);
    const float mg = fmaf(g2, gg, P.opsin_bias[1]);
    const float mb = fmaf(b2, gb, P.opsin_bias[2]);
    float lr = P.opsin_m[0] * mr, lg = P.opsin_m[3] * mr, lb = P.opsin_m[6] * mr;
    lr = fmaf(P.opsin_m[1], mg, lr); lg = fmaf(P.opsin_m[4], mg, lg); lb = fmaf(P.opsin_m[7], mg, lb);
    lr = fmaf(P.opsin_m[2], mb, lr); lg = fmaf(P.opsin_m[5], mb, lg); lb = fmaf(P.opsin_m[8], mb, lb);
    a = lr; b = lg; c3 = lb;
  }
  store_px<1>(P, out, out_row_stride, Y, X, (int)P.out_hh, a, b, c3);
}

// Noise planes (Random3Planes, lib/jxl/dec_noise.cc:45-110): per 256x256 tile of the output image a
// Xorshift128Plus with eight 128-bit states (lib/jxl/xorshift128plus-inl.h:31-91), seeded with the two frame
// indices and the tile origin, fills plane 0, then 1, then 2, row by row, 16 floats (eight 64-bit outputs) per
// step, "1.0 + 23 random mantissa bits".  The generator is sequential per tile: eight lanes carry the eight
// states of one tile, four tiles per warp.
__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__global__ void __launch_bounds__(32) noise_gen_kernel(float* __restrict__ planes, uint32_t W, uint32_t H, uint32_t visible,
                                                       uint32_t nonvisible) {
  const uint32_t lane = threadIdx.x & 7u;
  const uint32_t tiles_x = (W + 255u) / 256u, tiles_y = (H + 255u) / 256u;
  const uint32_t tile = blockIdx.x * 4u + (threadIdx.x >> 3);
  if (tile >= tiles_x * tiles_y) return;
  const uint32_t x0 = (tile % tiles_x) * 256u, y0 = (tile / tiles_x) * 256u;
  const uint32_t xs = min(256u, W - x0), ys = min(256u, H - y0);
  // state `lane` of the generator: s0[i] = SplitMix64^i(s0[0]), s1[i] likewise
  uint64_t s0 = splitmix64((((uint64_t)visible << 32) + nonvisible) + 0x9E3779B97F4A7C15ull);
  uint64_t s1 = splitmix64((((uint64_t)x0 << 32) + y0) + 0x9E3779B97F4A7C15ull);
  for (uint32_t i = 0; i < lane; i++) {
    s0 = splitmix64(s0);
    s1 = splitmix64(s1);
  }
  const size_t plane = (size_t)W * H;
#pragma unroll 1
  for (int p = 0; p < 3; p++)
#pragma unroll 1
    for (uint32_t y = 0; y < ys; y++) {
      float* row = planes + (size_t)p * plane + (size_t)(y0 + y) * W + x0;
      // entire batches while x + 16 < xs, then one more batch for the remaining (at most 16) pixels
#pragma unroll 1
      for (uint32_t x = 0;; x += 16) {
        uint64_t a = s0;
        const uint64_t b = s1;
        const uint64_t bits = a + b;
        s0 = b;
        a ^= a << 23;
        a ^= b ^ (a >> 18) ^ (b >> 5);
        s1 = a;
        const uint32_t xa = x + 2u * lane;
        if (xa < xs) row[xa] = __uint_as_float(((uint32_t)bits >> 9) | 0x3F800000u);
        if (xa + 1 < xs) row[xa + 1] = __uint_as_float(((uint32_t)(bits >> 32) >> 9) | 0x3F800000u);
        if (!(x + 16 < xs)) break;
      }
    }
}

// ---------------------------------------------------------------------------
// UpsamplingStage (lib/jxl/render_pipeline/stage_upsampling.cc:51-271; SURVEY.md §8f rank 4) fused with the
// stages PreparePipeline puts behind it (dec_cache.cc:216-330): XYB -> linear RGB [-> sRGB] -> output packing.
// `in`: the filtered XYB planes at the coded size ([3][ysize][xsize] f32, written by the filter chain run
// without its XYB stage).  One thread per OUTPUT pixel (X, Y): sub-pixel k = N*(Y%N) + X%N of input pixel
// (X/N, Y/N); 25 taps of the 5x5 window (mirrored about the coded size) in three accumulators in the
// reference's order (:246-262), clamped to the window's minimum / maximum (:152-206).
// ---------------------------------------------------------------------------
// ConvolveNoiseStage (stage_noise.cc:263-304) over the three generated planes, once per frame: 24 neighbours summed
// in the reference's order, 0.16 * sum - 3.84 * centre; borders mirrored about the output size.
__global__ void __launch_bounds__(256) noise_conv_kernel(const float* __restrict__ raw, float* __restrict__ conv, int OW, int OH) {
  const int X = blockIdx.x * 32 + (threadIdx.x & 31), Y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (X >= OW || Y >= OH) return;
  int cx[5], ry[5];
#pragma unroll
  for (int d = 0; d < 5; d++) {
    cx[d] = mirror_i(X + d - 2, OW);
    ry[d] = mirror_i(Y + d - 2, OH) * OW;
  }
  const float* p = raw + (size_t)blockIdx.z * OW * OH;
  float others = 0.0f;
#pragma unroll
  for (int i = 0; i < 5; i++) {
    others = others + __ldg(p + ry[0] + cx[i]);
    others = others + __ldg(p + ry[1] + cx[i]);
    others = others + __ldg(p + ry[3] + cx[i]);
    others = others + __ldg(p + ry[4] + cx[i]);
  }
  others = others + __ldg(p + ry[2] + cx[0]);
  others = others + __ldg(p + ry[2] + cx[1]);
  others = others + __ldg(p + ry[2] + cx[3]);
  others = others + __ldg(p + ry[2] + cx[4]);
  conv[((size_t)blockIdx.z * OH + Y) * OW + X] = fmaf(others, 0.16f, __ldg(p + ry[2] + cx[2]) * -3.84f);
}

__global__ void __launch_bounds__(256) upsample_kernel(const __grid_constant__ FrameDev P, const float* __restrict__ in,
                                                       char* __restrict__ out, size_t out_row_stride) {
  const int X = blockIdx.x * 32 + (threadIdx.x & 31), Y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (X >= (int)P.out_w || Y >= (int)P.out_hh) return;
  const int N = P.ups ? (int)P.ups : 1, W = (int)P.xsize, H = (int)P.ysize;
  if (N == 1) {  // no upsampling: the filtered planes are the stage's input as they are (noise-only frames)
    float a = __ldg(in + (size_t)Y * W + X), b = __ldg(in + (size_t)W * H + (size_t)Y * W + X),
          c3 = __ldg(in + 2 * (size_t)W * H + (size_t)Y * W + X);
    finish_px(P, out, out_row_stride, X, Y, a, b, c3);
    return;
  }
  const int x = X / N, y = Y / N;
  const float* k = P.ups_kernel + (N * (Y - y * N) + (X - x * N)) * 25;
  int cx[5], ry[5];
#pragma unroll
  for (int d = 0; d < 5; d++) {
    cx[d] = mirror_i(x + d - 2, W);
    ry[d] = mirror_i(y + d - 2, H) * W;
  }
  float kw[25];
#pragma unroll
  for (int i = 0; i < 25; i++) kw[i] = __ldg(k + i);
  float res[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float* p = in + (size_t)c * W * H;
    float v[25];
#pragma unroll
    for (int iy = 0; iy < 5; iy++)
#pragma unroll
      for (int ix = 0; ix < 5; ix++) v[5 * iy + ix] = __ldg(p + ry[iy] + cx[ix]);
    float mn = v[0], mx = v[0];
#pragma unroll
    for (int i = 1; i < 25; i++) {
      mn = fminf(mn, v[i]);
      mx = fmaxf(mx, v[i]);
    }
    float a0 = v[0] * kw[0], a1 = v[1] * kw[1], a2 = v[2] * kw[2];
#pragma unroll
    for (int i = 3; i < 24; i += 3) {
      a0 = fmaf(v[i], kw[i], a0);
      a1 = fmaf(v[i + 1], kw[i + 1], a1);
      a2 = fmaf(v[i + 2], kw[i + 2], a2);
    }
    a0 = fmaf(v[24], kw[24], a0);
    float r = (a1 + a2) + a0;
    r = r < mn ? mn : r;
    r = r > mx ? mx : r;
    res[c] = r;
  }
  finish_px(P, out, out_row_stride, X, Y, res[0], res[1], res[2]);
}

// The same stage with one thread per INPUT pixel: the 5x5 window of the three channels is loaded once (75 values
// in registers, plus its minima / maxima) and reused for the N x N outputs of the pixel, whose taps come from a
// shared-memory copy of the table -- upsample_kernel reloads the window for every output pixel (N^2 times).
template <int N>
__global__ void __launch_bounds__(256) upsample_in_kernel(const __grid_constant__ FrameDev P, const float* __restrict__ in,
                                                          char* __restrict__ out, size_t out_row_stride) {
  __shared__ float taps[N * N * 25];
  for (int i = threadIdx.x; i < N * N * 25; i += 256) taps[i] = __ldg(P.ups_kernel + i);
  __syncthreads();
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int W = (int)P.xsize, H = (int)P.ysize;
  if (x >= W || y >= H) return;
  int cx[5], ry[5];
#pragma unroll
  for (int d = 0; d < 5; d++) {
    cx[d] = mirror_i(x + d - 2, W);
    ry[d] = mirror_i(y + d - 2, H) * W;
  }
  float v[3][25], mn[3], mx[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float* p = in + (size_t)c * W * H;
#pragma unroll
    for (int iy = 0; iy < 5; iy++)
#pragma unroll
      for (int ix = 0; ix < 5; ix++) v[c][5 * iy + ix] = __ldg(p + ry[iy] + cx[ix]);
    mn[c] = mx[c] = v[c][0];
#pragma unroll
    for (int i = 1; i < 25; i++) {
      mn[c] = fminf(mn[c], v[c][i]);
      mx[c] = fmaxf(mx[c], v[c][i]);
    }
  }
#pragma unroll 1
  for (int oy = 0; oy < N; oy++) {
    const int Y = y * N + oy;
    if (Y >= (int)P.out_hh) break;
#pragma unroll 1
    for (int ox = 0; ox < N; ox++) {
      const int X = x * N + ox;
      if (X >= (int)P.out_w) break;
      const float* kw = taps + (N * oy + ox) * 25;
      float res[3];
#pragma unroll
      for (int c = 0; c < 3; c++) {
        float a0 = v[c][0] * kw[0], a1 = v[c][1] * kw[1], a2 = v[c][2] * kw[2];
#pragma unroll
        for (int i = 3; i < 24; i += 3) {
          a0 = fmaf(v[c][i], kw[i], a0);
          a1 = fmaf(v[c][i + 1], kw[i + 1], a1);
          a2 = fmaf(v[c][i + 2], kw[i + 2], a2);
        }
        a0 = fmaf(v[c][24], kw[24], a0);
        float r = (a1 + a2) + a0;
        r = r < mn[c] ? mn[c] : r;
        r = r > mx[c] ? mx[c] : r;
        res[c] = r;
      }
      finish_px(P, out, out_row_stride, X, Y, res[0], res[1], res[2]);
    }
  }
}

__global__ void __launch_bounds__(kFilterThreads) filter_kernel(const __grid_constant__ FrameDev P,
                                                               char* __restrict__ out,
                                                               size_t out_row_stride /*bytes*/) {
  extern __shared__ __align__(16) float fsm[];
  float* bufA = fsm;
  float* bufB = fsm + 3 * kTilePlane;
  const int tid = threadIdx.x;
  const int W = (int)P.xsize, H = (int)P.ysize;
  const int tile_x = blockIdx.x * kTW;
  const int tile_y = (int)P.band_y0 + blockIdx.y * kTH;
  const uint32_t mask = P.stage_mask;
  const int halo = ((mask & 1) ? 1 : 0) + ((mask & 2) ? 3 : 0) + ((mask & 4) ? 2 : 0) + ((mask & 8) ? 1 : 0);
  TileGeom G;
  G.x0 = tile_x - halo;
  G.y0 = tile_y - halo;
  G.W = W;
  G.H = H;
  const int SW = kTW + 2 * halo, SH = kTH + 2 * halo;
  G.edge = (G.x0 < 0) || (G.y0 < 0) || (G.x0 + SW > W) || (G.y0 + SH > H);
  // ---- load (positions inside the image only) ----
  for (int c = 0; c < 3; c++) {
    const float* src = P.xyb + (size_t)c * P.plane_stride;
    for (int i = tid; i < SH * SW; i += kFilterThreads) {
      const int ty = i / SW, tx = i % SW;
      const int y = G.y0 + ty, x = G.x0 + tx;
      if (y >= 0 && y < H && x >= 0 && x < W) bufA[c * kTilePlane + ty * kSP + tx] = src[(size_t)y * P.row_stride + x];
    }
  }
  __syncthreads();
  float* cur = bufA;
  float* nxt = bufB;
  int m = 0;  // margin already consumed
  // ---- Gaborish (stage_gaborish.cc:56-100) ----
  if (mask & 1) {
    m += 1;
    const int rw = SW - 2 * m, rh = SH - 2 * m;
    for (int i = tid; i < rw * rh; i += kFilterThreads) {
      const int ty = m + i / rw, tx = m + i % rw;
      const int y = G.y0 + ty, x = G.x0 + tx;
      if (y < 0 || y >= H || x < 0 || x >= W) continue;
      const int o_t = G.at(ty - 1, tx), o_b = G.at(ty + 1, tx), o_l = G.at(ty, tx - 1), o_r = G.at(ty, tx + 1);
      const int o_tl = G.at(ty - 1, tx - 1), o_tr = G.at(ty - 1, tx + 1);
      const int o_bl = G.at(ty + 1, tx - 1), o_br = G.at(ty + 1, tx + 1);
      const int o_c = ty * kSP + tx;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float* p = cur + c * kTilePlane;
        const float sum1 = (p[o_l] + p[o_r]) + (p[o_t] + p[o_b]);
        const float sum2 = (p[o_tl] + p[o_tr]) + (p[o_bl] + p[o_br]);
        nxt[c * kTilePlane + o_c] = fmaf(sum2, P.gab_w[3 * c + 2], fmaf(sum1, P.gab_w[3 * c + 1], p[o_c] * P.gab_w[3 * c]));
      }
    }
    __syncthreads();
    float* t = cur; cur = nxt; nxt = t;
  }
  // ---- EPF passes (stage_epf.cc) ----
  const float kMinSigma = -3.90524291751269967465540850526868f;
#pragma unroll 1
  for (int pass = 0; pass < 3; pass++) {
    if (!(mask & (2u << pass))) continue;
    m += (pass == 0) ? 3 : (pass == 1 ? 2 : 1);
    const int rw = SW - 2 * m, rh = SH - 2 * m;
    const float sm_ = P.epf_sm[pass];
    const float bsm = sm_ * P.epf_border_mul;
    for (int i = tid; i < rw * rh; i += kFilterThreads) {
      const int ty = m + i / rw, tx = m + i % rw;
      const int y = G.y0 + ty, x = G.x0 + tx;
      if (y < 0 || y >= H || x < 0 || x >= W) continue;
      const int o_c = ty * kSP + tx;
      const float s = P.sigma[(size_t)(y >> 3) * P.xb + (x >> 3)];
      const float* pX = cur;
      const float* pY = cur + kTilePlane;
      const float* pB = cur + 2 * kTilePlane;
      if (s < kMinSigma) {
        nxt[o_c] = pX[o_c];
        nxt[kTilePlane + o_c] = pY[o_c];
        nxt[2 * kTilePlane + o_c] = pB[o_c];
        continue;
      }
      const int iy = y & 7, ix = x & 7;
      const float vsm = (iy == 0 || iy == 7 || ix == 0 || ix == 7) ? bsm : sm_;
      const float inv_sigma = s * vsm;
      float w = 1.0f, X = pX[o_c], Y = pY[o_c], B = pB[o_c];
      if (pass == 0) {
        // 12 neighbours, SAD over the 5-pixel plus window (stage_epf.cc:134-166)
        const int dy12[12] = {-2, -1, -1, -1, 0, 0, 0, 0, 1, 1, 1, 2};
        const int dx12[12] = {0, -1, 0, 1, -2, -1, 1, 2, -1, 0, 1, 0};
        const int py5[5] = {0, -1, 0, 1, 0};
        const int px5[5] = {0, 0, -1, 0, 1};
        float sads[12];
#pragma unroll
        for (int k = 0; k < 12; k++) sads[k] = 0.0f;
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float* p = cur + c * kTilePlane;
          const float scale = P.epf_scale[c];
#pragma unroll
          for (int k = 0; k < 12; k++) {
            float sad = 0.0f;
#pragma unroll
            for (int o = 0; o < 5; o++) {
              const float r11 = p[G.at(ty + py5[o], tx + px5[o])];
              const float c11 = p[G.at(ty + dy12[k] + py5[o], tx + dx12[k] + px5[o])];
              sad = sad + fabsf(r11 - c11);
            }
            sads[k] = fmaf(sad, scale, sads[k]);
          }
        }
#pragma unroll
        for (int k = 0; k < 12; k++) {
          const float wt = epf_weight(sads[k], inv_sigma);
          const int o = G.at(ty + dy12[k], tx + dx12[k]);
          w = w + wt;
          X = fmaf(wt, pX[o], X);
          Y = fmaf(wt, pY[o], Y);
          B = fmaf(wt, pB[o], B);
        }
      } else if (pass == 1) {
        // 4 neighbours, plus-window SADs with shared terms (stage_epf.cc:278-336)
        const int o20 = G.at(ty - 2, tx), o21 = G.at(ty - 1, tx), o11 = G.at(ty - 1, tx - 1), o31 = G.at(ty - 1, tx + 1);
        const int o02 = G.at(ty, tx - 2), o12 = G.at(ty, tx - 1), o32 = G.at(ty, tx + 1), o42 = G.at(ty, tx + 2);
        const int o13 = G.at(ty + 1, tx - 1), o23 = G.at(ty + 1, tx), o33 = G.at(ty + 1, tx + 1), o24 = G.at(ty + 2, tx);
        float sad0 = 0.0f, sad1 = 0.0f, sad2 = 0.0f, sad3 = 0.0f;
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float* p = cur + c * kTilePlane;
          const float p20 = p[o20], p21 = p[o21], p11 = p[o11], p31 = p[o31];
          const float p02 = p[o02], p12 = p[o12], p22 = p[o_c], p32 = p[o32], p42 = p[o42];
          const float p13 = p[o13], p23 = p[o23], p33 = p[o33], p24 = p[o24];
          float t;
          float sad0c = fabsf(p20 - p21);
          float sad1c = fabsf(p11 - p21);
          float sad2c = fabsf(p31 - p21);
          sad1c = sad1c + fabsf(p02 - p12);
          sad0c = sad0c + fabsf(p11 - p12);
          t = fabsf(p12 - p22);
          sad1c = sad1c + t;
          sad2c = sad2c + t;
          t = fabsf(p22 - p21);
          float sad3c = t;
          sad0c = sad0c + t;
          sad0c = sad0c + fabsf(p31 - p32);
          t = fabsf(p22 - p32);
          sad1c = sad1c + t;
          sad2c = sad2c + t;
          sad2c = sad2c + fabsf(p42 - p32);
          sad3c = sad3c + fabsf(p13 - p12);
          t = fabsf(p22 - p23);
          sad0c = sad0c + t;
          sad3c = sad3c + t;
          sad1c = sad1c + fabsf(p13 - p23);
          sad2c = sad2c + fabsf(p33 - p23);
          sad3c = sad3c + fabsf(p33 - p32);
          sad3c = sad3c + fabsf(p24 - p23);
          const float scale = P.epf_scale[c];
          sad0 = fmaf(sad0c, scale, sad0);
          sad1 = fmaf(sad1c, scale, sad1);
          sad2 = fmaf(sad2c, scale, sad2);
          sad3 = fmaf(sad3c, scale, sad3);
        }
        const float sd[4] = {sad0, sad1, sad2, sad3};
        const int on[4] = {o21, o12, o32, o23};
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const float wt = epf_weight(sd[k], inv_sigma);
          w = w + wt;
          X = fmaf(wt, pX[on[k]], X);
          Y = fmaf(wt, pY[on[k]], Y);
          B = fmaf(wt, pB[on[k]], B);
        }
      } else {
        // 4 neighbours, single-pixel 3-channel SAD (stage_epf.cc:395-413)
        const float rx = X, ry = Y, rb = B;
        const int on[4] = {G.at(ty - 1, tx), G.at(ty, tx - 1), G.at(ty, tx + 1), G.at(ty + 1, tx)};
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const float cx = pX[on[k]], cy = pY[on[k]], cb = pB[on[k]];
          float sad = fabsf(cx - rx) * P.epf_scale[0];
          sad = fmaf(fabsf(cy - ry), P.epf_scale[1], sad);
          sad = fmaf(fabsf(cb - rb), P.epf_scale[2], sad);
          const float wt = epf_weight(sad, inv_sigma);
          w = w + wt;
          X = fmaf(wt, cx, X);
          Y = fmaf(wt, cy, Y);
          B = fmaf(wt, cb, B);
        }
      }
      const float inv_w = 1.0f / w;
      nxt[o_c] = X * inv_w;
      nxt[kTilePlane + o_c] = Y * inv_w;
      nxt[2 * kTilePlane + o_c] = B * inv_w;
    }
    __syncthreads();
    float* t = cur; cur = nxt; nxt = t;
  }
  // ---- XYB -> linear RGB (dec_xyb-inl.h:38-86) + store ----
  const int band_h = (int)P.out_h;
  for (int i = tid; i < kTW * kTH; i += kFilterThreads) {
    const int ty = halo + i / kTW, tx = halo + i % kTW;
    const int y = G.y0 + ty, x = G.x0 + tx;
    if (y >= (int)P.band_y1 || x >= W) continue;
    const int o_c = ty * kSP + tx;
    float a = cur[o_c], b = cur[kTilePlane + o_c], c3 = cur[2 * kTilePlane + o_c];
    if ((mask & 16) && P.ycbcr) {
      ycbcr_px(a, b, c3);
    } else if (mask & 16) {
      float gr = b + a, gg = b - a, gb = c3;
      gr = gr - P.opsin_cbrt[0];
      gg = gg - P.opsin_cbrt[1];
      gb = gb - P.opsin_cbrt[2];
      const float r2 = gr * gr, g2 = gg * gg, b2 = gb * gb;
      const float mr = fmaf(r2, gr, P.opsin_bias[0]);
      const float mg = fmaf(g2, gg, P.opsin_bias[1]);
      const float mb = fmaf(b2, gb, P.opsin_bias[2]);
      float lr = P.opsin_m[0] * mr, lg = P.opsin_m[3] * mr, lb = P.opsin_m[6] * mr;
      lr = fmaf(P.opsin_m[1], mg, lr); lg = fmaf(P.opsin_m[4], mg, lg); lb = fmaf(P.opsin_m[7], mg, lb);
      lr = fmaf(P.opsin_m[2], mb, lr); lg = fmaf(P.opsin_m[5], mb, lg); lb = fmaf(P.opsin_m[8], mb, lb);
      a = lr; b = lg; c3 = lb;
    }
    store_px<1>(P, out, out_row_stride, y - (int)P.out_y0, x, band_h, a, b, c3);
  }
}

#endif  // JXLB_STRIP_TU

}  // namespace jxlb

// ===========================================================================
// filter v2: row-streaming strip kernel (the fast path for the stage chains real
// frames use).  One CTA owns a vertical strip of kStripThreads columns (output
// columns + the chain's halo on both sides) and marches down the rows of its
// segment.  Every enabled stage keeps a small ring of its INPUT rows in shared
// memory and produces exactly one row per step; stage k works on the row that
// became computable after the previous step, so one __syncthreads() per step
// orders everything.  No vertical halo is recomputed inside a segment, the
// horizontal halo costs 2*H of 256 lanes, and nothing but the final RGB row is
// written to global memory.
//
// The row loop has two bodies generated from the same source: the generic one
// (row-range predicates, row mirroring, lane-range predicates) runs the few
// steps of pipeline fill / drain and everything near the top or bottom image
// edge; the STEADY one assumes every stage has a valid, unmirrored row this
// step and lets out-of-range lanes compute garbage that nobody reads (the
// shared-memory rings are padded so their neighbour reads stay in bounds).
//
// Arithmetic (operation order, FMAs) is identical to filter_kernel above and to
// the reference stages it cites.
// ===========================================================================
namespace jxlb {

template <int V>
using IC = std::integral_constant<int, V>;

constexpr int kStripThreads = 256;
constexpr int kStripPad = 4;  // floats of padding before/after the rings

template <uint32_t MASK>
struct StripCfg {
  static constexpr bool G = (MASK & 1) != 0, E0 = (MASK & 2) != 0, E1 = (MASK & 4) != 0, E2 = (MASK & 8) != 0;
  static constexpr bool XYB = (MASK & 16) != 0;
  static constexpr int H = (G ? 1 : 0) + (E0 ? 3 : 0) + (E1 ? 2 : 0) + (E2 ? 1 : 0);
  // ring sizes (rows, power of two >= 2*border+2) of each stage's input; 0 when absent
  static constexpr int NG = G ? 4 : 0, N0 = E0 ? 8 : 0, N1 = E1 ? 8 : 0, N2 = E2 ? 4 : 0;
  static constexpr int kRows = NG + N0 + N1 + N2;
  // Chains with an EPF pass run those passes on a PERMUTATION of the strip's 32 block columns, the blocks whose
  // sigma engages the filter first (see filter_strip_body): the strip then starts on a block boundary.
  static constexpr bool kCompact = E0 || E1 || E2;
  static constexpr int LEAD = kCompact ? 8 : H;  // strip column of the first output column
  static constexpr size_t kListBytes = kCompact ? 4 * 32 * 8 : 0;  // [4 block rows][32] permutation + sigma
  static constexpr size_t kSmemBytes =
      ((size_t)(kRows ? kRows : 1) * 3 * kStripThreads + 2 * kStripPad) * sizeof(float) + kListBytes;
  static constexpr int kOutCols = kStripThreads - 2 * LEAD;
};

__device__ __forceinline__ float* ring_row(float* ring, int n, int r, int c) {
  return ring + ((r & (n - 1)) * 3 + c) * kStripThreads;
}

template <uint32_t MASK, bool EDGE, bool REPL, int OUTK>
__device__ __forceinline__ void filter_strip_body(const FrameDev& P, char* __restrict__ out,
                                                  size_t out_row_stride /*bytes*/, int x0, int y_begin, int y_end,
                                                  float* smem) {
  using C = StripCfg<MASK>;
  constexpr int H = C::H;
  const int t = threadIdx.x;
  const int W = (int)P.xsize, HI = (int)P.ysize;
  constexpr int LEAD = C::LEAD;
  const int xs0 = x0 - LEAD;  // image column of strip column 0 (a multiple of 8 when the chain has an EPF pass)
  const int x = xs0 + t;      // image column of this thread
  const bool xin = x >= 0 && x < W;
  const int xs = min(max(x, 0), W - 1) >> 3;  // sigma column (clamped: garbage lanes stay in bounds)
  // strip-relative indices of the horizontal neighbours x-3 .. x+3 (mirrored at the image edge)
  int cn[7];
#pragma unroll
  for (int d = -3; d <= 3; d++) cn[d + 3] = EDGE ? (mirror_i(x + d, W) - xs0) : (t + d);
#ifdef JXLB_EMU_CLAMP_GARBAGE_LANES
  // ThreadSanitizer build of tests/emu only: the outermost H lanes of a strip compute values nobody reads
  // and, with cn = t + d, read a few floats of the neighbouring ring row while its owner writes them -- a
  // deliberate, harmless overlap (the rings are padded for it) that would drown real reports.  Keeping
  // those lanes inside their own row changes no lane whose result is used.
  for (int k = 0; k < 7; k++) cn[k] = min(max(cn[k], 0), kStripThreads - 1);
#endif
  // Mirror() (lib/jxl/image_ops.h:184-196) reflects repeatedly: images lower than a stage's border
  auto mrow = [&](int r) { return mirror_i(r, HI); };

  float* ringG = smem + kStripPad;
  float* ring0 = ringG + C::NG * 3 * kStripThreads;
  float* ring1 = ring0 + C::N0 * 3 * kStripThreads;
  float* ring2 = ring1 + C::N1 * 3 * kStripThreads;
  // EPF block permutation: for each of the (up to four) block rows in flight, the strip's 32 block columns
  // ordered "sigma engages the filter" first, and the blocks' inverse sigmas
  int* permv = reinterpret_cast<int*>(ring2 + C::N2 * 3 * kStripThreads + kStripPad);
  float* sigv = reinterpret_cast<float*>(permv + 4 * 32);

  // halo consumed after each stage: that stage computes lanes [h, 256 - h)
  constexpr int hG = C::G ? 1 : 0;
  constexpr int h0 = hG + (C::E0 ? 3 : 0);
  constexpr int h1 = h0 + (C::E1 ? 2 : 0);
  constexpr int h2 = h1 + (C::E2 ? 1 : 0);
  static_assert(h2 == H, "halo bookkeeping");
  // a stage whose output still feeds `rem` rows of halo produces rows [y_begin-rem, y_end+rem) ∩ image
  auto lo = [&](int rem) { return max(0, y_begin - rem); };
  auto hi = [&](int rem) { return min(HI, y_end + rem); };

  const bool xborder = ((x & 7) == 0 || (x & 7) == 7);  // (compact chains: the same for every column a lane is given)
  const int band_h = (int)P.out_h;

  // Final step of the chain: XYB -> linear RGB (dec_xyb-inl.h:38-86) and the global store.
  auto emit = [&](int r, int col, float a, float b, float c3) {
    const int xe = xs0 + col;
    if (!(col >= LEAD && col < kStripThreads - LEAD && xe < W)) return;
    if (C::XYB && !P.skip_xyb && P.ycbcr) {
      ycbcr_px(a, b, c3);
    } else if (C::XYB && !P.skip_xyb) {
      float gr = b + a, gg = b - a, gb = c3;
      gr = gr - P.opsin_cbrt[0];
      gg = gg - P.opsin_cbrt[1];
      gb = gb - P.opsin_cbrt[2];
      const float r2 = gr * gr, g2 = gg * gg, b2 = gb * gb;
      const float mr = fmaf(r2, gr, P.opsin_bias[0]);
      const float mg = fmaf(g2, gg, P.opsin_bias[1]);
      const float mb = fmaf(b2, gb, P.opsin_bias[2]);
      float lr = P.opsin_m[0] * mr, lg = P.opsin_m[3] * mr, lb = P.opsin_m[6] * mr;
      lr = fmaf(P.opsin_m[1], mg, lr); lg = fmaf(P.opsin_m[4], mg, lg); lb = fmaf(P.opsin_m[7], mg, lb);
      lr = fmaf(P.opsin_m[2], mb, lr); lg = fmaf(P.opsin_m[5], mb, lg); lb = fmaf(P.opsin_m[8], mb, lb);
      a = lr; b = lg; c3 = lb;
    }
    store_px<OUTK>(P, out, out_row_stride, r - (int)P.out_y0, xe, band_h, a, b, c3);
  };
  // cumulative delays (steps between loading row r and the stage producing row r)
  constexpr int dG = C::G ? 2 : 0;
  constexpr int d0 = dG + (C::E0 ? 4 : 0);
  constexpr int d1 = d0 + (C::E1 ? 3 : 0);
  constexpr int d2 = d1 + (C::E2 ? 2 : 0);
  const int r_in_lo = lo(H), r_in_hi = hi(H);
  const int r_end = hi(0) + d2;  // after this many input-row steps the last output row is out
  const float kMinSigma = -3.90524291751269967465540850526868f;

  // row r_in_lo is fetched up front, every later row one step ahead of its use
  float pre_a = 0.0f, pre_b = 0.0f, pre_c = 0.0f;
  if (r_in_lo < r_in_hi && xin) {
    const size_t off = (size_t)r_in_lo * P.row_stride + x;
    pre_a = __ldg(P.xyb + off);
    pre_b = __ldg(P.xyb + P.plane_stride + off);
    pre_c = __ldg(P.xyb + 2 * P.plane_stride + off);
  }

  // inverse sigma of each EPF stage's next row, fetched one step ahead as well.  A stage's first
  // produced row is max(0, y_begin - rem) (its `lo`), reached at step lo + delay.
  // ---- EPF block permutation ----
  // The filter is skipped where a block's sigma is below kMinSigma (stage_epf.cc:121-128) -- on typical frames
  // most blocks.  With one column per lane a warp spans four blocks and runs the EPF arithmetic as soon as one
  // of them is engaged, three quarters of its lanes masked off.  Instead every EPF pass works on a permutation
  // of the strip's 32 block columns, engaged blocks first: lane t handles column 8 * perm[t / 8] + t % 8, so
  // the engaged blocks fill whole warps and the remaining warps only copy their pixels through.  The
  // permutation of a block row is built by warp 0 when the loader reaches the row above it.
  auto build_lists = [&](int row) {
    if constexpr (C::kCompact) {
      if (t < 32) {
        const int br = row >> 3;
        const int bx = (xs0 >> 3) + t;
        float sv = -1e30f;  // outside the image: never engaged
        if (bx >= 0 && bx < (int)P.xb) sv = __ldg(P.sigma + (size_t)br * P.xb + bx);
        const bool act = !(sv < kMinSigma);
        const unsigned m = __ballot_sync(0xffffffffu, act);
        const unsigned lt = (1u << t) - 1u;
        const int pos = act ? __popc(m & lt) : __popc(m) + __popc(~m & lt);
        permv[(br & 3) * 32 + pos] = t;  // (rotating the first engaged warp per CTA / block row measured 4 % slower)
        sigv[(br & 3) * 32 + t] = sv;
      }
    }
  };
  // per EPF pass: the column this lane handles in the pass's current block row, that block's inverse sigma,
  // and (edge strips) the mirrored strip columns col-3 .. col+3
  int colE0 = t, colE1 = t, colE2 = t;
  float sgE0 = 0.0f, sgE1 = 0.0f, sgE2 = 0.0f;
  int cnE0[7], cnE1[7], cnE2[7];
#pragma unroll
  for (int k = 0; k < 7; k++) cnE0[k] = cnE1[k] = cnE2[k] = cn[k];
  auto load_sel = [&](int r, int& col, float& sg, int* cnk) {
    const int slot = (r >> 3) & 3;
    const int b = permv[slot * 32 + (t >> 3)];
    col = 8 * b + (t & 7);
    sg = sigv[slot * 32 + b];
    if constexpr (EDGE) {
#pragma unroll
      for (int d = -3; d <= 3; d++) cnk[d + 3] = mirror_i(xs0 + col + d, W) - xs0;
    }
#ifdef JXLB_EMU_CLAMP_GARBAGE_LANES
    for (int k = 0; k < 7; k++) cnk[k] = min(max(EDGE ? cnk[k] : col + k - 3, 0), kStripThreads - 1);
#endif
  };
  // does the lane produce column `col` of a pass whose cumulative halo is `h`?
  auto lane_run = [&](auto steady_tag, int col, int h) {
    constexpr bool ST = decltype(steady_tag)::value;
    if constexpr (ST && !EDGE) return true;
    const int xc = xs0 + col;
    bool ok = xc >= 0 && xc < W;
    if constexpr (!ST) ok = ok && col >= h && col < kStripThreads - h;
    return ok;
  };
  if (r_in_lo < r_in_hi) build_lists(r_in_lo);

  // One pipeline step.
  //   ST (steady): every stage has an in-range, unmirrored row; lanes are not range-checked (only
  //     `xin` in edge strips, where garbage lanes would read global memory).
  //   J >= 0 (aligned): rin == 8*m + J, so every ring slot (row & (n-1)) is a compile-time constant
  //     and shared-memory addresses are `lane base + immediate`; J == -1: slots computed at run time.
  auto step = [&](auto steady_tag, auto jtag, int rin) {
    constexpr bool ST = decltype(steady_tag)::value;
    constexpr int J = decltype(jtag)::value;
    static_assert(J < 0 || ST, "aligned steps are steady steps");
    auto mr = [&](int r) { return ST ? r : mrow(r); };
    // channel-0 row pointer of ring row (rin + dk); r_dyn is that row (mirrored in generic mode)
    auto RP = [&](float* ring, auto ntag, auto dktag, int r_dyn) -> float* {
      constexpr int n = decltype(ntag)::value;
      constexpr int dk = decltype(dktag)::value;
      if constexpr (J >= 0) return ring + ((((J + dk) % n + n) % n) * 3) * kStripThreads;
      else return ring + ((r_dyn & (n - 1)) * 3) * kStripThreads;
    };
    // Hand a stage's result (row rin - D) to the next stage's ring, or emit it after the last stage.
    // `which`: 0 = loader output, 1 = Gaborish, 2 = EPF0, 3 = EPF1, 4 = EPF2.
    auto deliver = [&](auto which_tag, int r, int col, float X, float Y, float B) {
      constexpr int which = decltype(which_tag)::value;
      constexpr int D = which == 0 ? 0 : (which == 1 ? dG : (which == 2 ? d0 : (which == 3 ? d1 : d2)));
      constexpr bool toG = which < 1 && C::G;
      constexpr bool to0 = !toG && which < 2 && C::E0;
      constexpr bool to1 = !toG && !to0 && which < 3 && C::E1;
      constexpr bool to2 = !toG && !to0 && !to1 && which < 4 && C::E2;
      float* dst = nullptr;
      if constexpr (toG) dst = RP(ringG, IC<C::NG ? C::NG : 1>(), IC<-D>(), r);
      else if constexpr (to0) dst = RP(ring0, IC<C::N0 ? C::N0 : 1>(), IC<-D>(), r);
      else if constexpr (to1) dst = RP(ring1, IC<C::N1 ? C::N1 : 1>(), IC<-D>(), r);
      else if constexpr (to2) dst = RP(ring2, IC<C::N2 ? C::N2 : 1>(), IC<-D>(), r);
      if constexpr (toG || to0 || to1 || to2) {
        dst[col] = X;
        dst[kStripThreads + col] = Y;
        dst[2 * kStripThreads + col] = B;
      } else {
        emit(r, col, X, Y, B);
      }
    };
    const bool lane_ok = (ST && !EDGE) ? true : xin;
    // ---- loader: XYB row rin was fetched during the previous step (its latency hid behind that
    // step's arithmetic); hand it on and start fetching row rin + 1 ----
    if ((ST || rin < r_in_hi) && xin) deliver(IC<0>(), rin, t, pre_a, pre_b, pre_c);
    if constexpr (C::kCompact) {  // the block row that starts with the next input row
      if ((J >= 0 ? J == 7 : ((rin + 1) & 7) == 0) && rin + 1 < r_in_hi) build_lists(rin + 1);
    }
    if (rin + 1 < r_in_hi && xin) {
      const size_t off = (size_t)(rin + 1) * P.row_stride + x;
      pre_a = __ldg(P.xyb + off);
      pre_b = __ldg(P.xyb + P.plane_stride + off);
      pre_c = __ldg(P.xyb + 2 * P.plane_stride + off);
    }
    // ---- Gaborish (stage_gaborish.cc:56-100) ----
    if constexpr (C::G) {
      const int r = rin - dG;
      if ((ST || (r >= lo(H - hG) && r < hi(H - hG) && t >= hG && t < kStripThreads - hG)) && lane_ok) {
        const float* pT0 = RP(ringG, IC<C::NG>(), IC<-dG - 1>(), mr(r - 1));
        const float* pM0 = RP(ringG, IC<C::NG>(), IC<-dG>(), r);
        const float* pB0 = RP(ringG, IC<C::NG>(), IC<-dG + 1>(), mr(r + 1));
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float* pT = pT0 + c * kStripThreads;
          const float* pM = pM0 + c * kStripThreads;
          const float* pB = pB0 + c * kStripThreads;
          const float sum1 = (pM[cn[2]] + pM[cn[4]]) + (pT[t] + pB[t]);
          const float sum2 = (pT[cn[2]] + pT[cn[4]]) + (pB[cn[2]] + pB[cn[4]]);
          v[c] = fmaf(sum2, P.gab_w[3 * c + 2], fmaf(sum1, P.gab_w[3 * c + 1], pM[t] * P.gab_w[3 * c]));
        }
        deliver(IC<1>(), r, t, v[0], v[1], v[2]);
      }
    }
    // ---- EPF0 (stage_epf.cc:54-193) ----
    if constexpr (C::E0) {
      const int r = rin - d0;
      const bool row_on = ST || (r >= lo(H - h0) && r < hi(H - h0));
      if (row_on && !(J >= 0 && ((J - d0) & 7) != 0)) load_sel(r, colE0, sgE0, cnE0);
      const int col = colE0;
      const int* cnk = cnE0;
      if (row_on && lane_run(steady_tag, col, h0)) {
        const float s = sgE0;
        const float* rows[7];
        rows[0] = RP(ring0, IC<C::N0>(), IC<-d0 - 3>(), mr(r - 3));
        rows[1] = RP(ring0, IC<C::N0>(), IC<-d0 - 2>(), mr(r - 2));
        rows[2] = RP(ring0, IC<C::N0>(), IC<-d0 - 1>(), mr(r - 1));
        rows[3] = RP(ring0, IC<C::N0>(), IC<-d0>(), r);
        rows[4] = RP(ring0, IC<C::N0>(), IC<-d0 + 1>(), mr(r + 1));
        rows[5] = RP(ring0, IC<C::N0>(), IC<-d0 + 2>(), mr(r + 2));
        rows[6] = RP(ring0, IC<C::N0>(), IC<-d0 + 3>(), mr(r + 3));
        float X = rows[3][col];
        float Y = rows[3][kStripThreads + col];
        float B = rows[3][2 * kStripThreads + col];
        if (!(s < kMinSigma)) {
          const int iy = r & 7;
          const float sm_ = P.epf_sm[0];
          const float vsm = (iy == 0 || iy == 7 || xborder) ? sm_ * P.epf_border_mul : sm_;
          const float inv_sigma = s * vsm;
          const int dy12[12] = {-2, -1, -1, -1, 0, 0, 0, 0, 1, 1, 1, 2};
          const int dx12[12] = {0, -1, 0, 1, -2, -1, 1, 2, -1, 0, 1, 0};
          const int py5[5] = {0, -1, 0, 1, 0};
          const int px5[5] = {0, 0, -1, 0, 1};
          float sads[12];
#pragma unroll
          for (int k = 0; k < 12; k++) sads[k] = 0.0f;
          float nbv[3][12];
#pragma unroll
          for (int c = 0; c < 3; c++) {
            // the 25 pixels of the radius-3 diamond, in registers
            float v[7][7];
#pragma unroll
            for (int a = 0; a < 7; a++)
#pragma unroll
              for (int b = 0; b < 7; b++)
                if ((a > 3 ? a - 3 : 3 - a) + (b > 3 ? b - 3 : 3 - b) <= 3)
                  v[a][b] = rows[a][c * kStripThreads + (EDGE ? cnk[b] : col + b - 3)];
            const float scale = P.epf_scale[c];
#pragma unroll
            for (int k = 0; k < 12; k++) {
              float sad = 0.0f;
#pragma unroll
              for (int o = 0; o < 5; o++) {
                // |a-b| == |b-a| exactly: always subtract in (row, column) order so that the 60
                // terms collapse to the ~32 distinct pixel pairs under common-subexpression elimination
                const int a0 = 3 + py5[o], b0 = 3 + px5[o];
                const int a1 = a0 + dy12[k], b1 = b0 + dx12[k];
                const bool sw = (a1 < a0) || (a1 == a0 && b1 < b0);
                const float lhs = sw ? v[a1][b1] : v[a0][b0];
                const float rhs = sw ? v[a0][b0] : v[a1][b1];
                sad = sad + fabsf(lhs - rhs);
              }
              sads[k] = fmaf(sad, scale, sads[k]);
              nbv[c][k] = v[3 + dy12[k]][3 + dx12[k]];
            }
          }
          float w = 1.0f;
#pragma unroll
          for (int k = 0; k < 12; k++) {
            const float wt = epf_weight(sads[k], inv_sigma);
            w = w + wt;
            X = fmaf(wt, nbv[0][k], X);
            Y = fmaf(wt, nbv[1][k], Y);
            B = fmaf(wt, nbv[2][k], B);
          }
          const float inv_w = 1.0f / w;
          X = X * inv_w; Y = Y * inv_w; B = B * inv_w;
        }
        deliver(IC<2>(), r, col, X, Y, B);
      }
    }
    // ---- EPF1 (stage_epf.cc:197-379) ----
    if constexpr (C::E1) {
      const int r = rin - d1;
      const bool row_on = ST || (r >= lo(H - h1) && r < hi(H - h1));
      if (row_on && !(J >= 0 && ((J - d1) & 7) != 0)) load_sel(r, colE1, sgE1, cnE1);
      const int col = colE1;
      const int* cnk = cnE1;
      auto CC = [&](int d) { return EDGE ? cnk[d + 3] : col + d; };
      if (row_on && lane_run(steady_tag, col, h1)) {
        const float s = sgE1;
        const float* q2x = RP(ring1, IC<C::N1>(), IC<-d1>(), r);
        float X = q2x[col];
        float Y = q2x[kStripThreads + col];
        float B = q2x[2 * kStripThreads + col];
        if (!(s < kMinSigma)) {
          const int iy = r & 7;
          const float sm_ = P.epf_sm[1];
          const float vsm = (iy == 0 || iy == 7 || xborder) ? sm_ * P.epf_border_mul : sm_;
          const float inv_sigma = s * vsm;
          const float* q0x = RP(ring1, IC<C::N1>(), IC<-d1 - 2>(), mr(r - 2));
          const float* q1x = RP(ring1, IC<C::N1>(), IC<-d1 - 1>(), mr(r - 1));
          const float* q3x = RP(ring1, IC<C::N1>(), IC<-d1 + 1>(), mr(r + 1));
          const float* q4x = RP(ring1, IC<C::N1>(), IC<-d1 + 2>(), mr(r + 2));
          float sad0 = 0.0f, sad1 = 0.0f, sad2 = 0.0f, sad3 = 0.0f;
          float nb[3][4];  // neighbour pixels N, W, E, S per channel
#pragma unroll
          for (int c = 0; c < 3; c++) {
            const float* q0 = q0x + c * kStripThreads;
            const float* q1 = q1x + c * kStripThreads;
            const float* q2 = q2x + c * kStripThreads;
            const float* q3 = q3x + c * kStripThreads;
            const float* q4 = q4x + c * kStripThreads;
            const float p20 = q0[col], p11 = q1[CC(-1)], p21 = q1[col], p31 = q1[CC(1)];
            const float p02 = q2[CC(-2)], p12 = q2[CC(-1)], p22 = q2[col], p32 = q2[CC(1)], p42 = q2[CC(2)];
            const float p13 = q3[CC(-1)], p23 = q3[col], p33 = q3[CC(1)], p24 = q4[col];
            nb[c][0] = p21; nb[c][1] = p12; nb[c][2] = p32; nb[c][3] = p23;
            float tt;
            float sad0c = fabsf(p20 - p21);
            float sad1c = fabsf(p11 - p21);
            float sad2c = fabsf(p31 - p21);
            sad1c = sad1c + fabsf(p02 - p12);
            sad0c = sad0c + fabsf(p11 - p12);
            tt = fabsf(p12 - p22);
            sad1c = sad1c + tt;
            sad2c = sad2c + tt;
            tt = fabsf(p22 - p21);
            float sad3c = tt;
            sad0c = sad0c + tt;
            sad0c = sad0c + fabsf(p31 - p32);
            tt = fabsf(p22 - p32);
            sad1c = sad1c + tt;
            sad2c = sad2c + tt;
            sad2c = sad2c + fabsf(p42 - p32);
            sad3c = sad3c + fabsf(p13 - p12);
            tt = fabsf(p22 - p23);
            sad0c = sad0c + tt;
            sad3c = sad3c + tt;
            sad1c = sad1c + fabsf(p13 - p23);
            sad2c = sad2c + fabsf(p33 - p23);
            sad3c = sad3c + fabsf(p33 - p32);
            sad3c = sad3c + fabsf(p24 - p23);
            const float scale = P.epf_scale[c];
            sad0 = fmaf(sad0c, scale, sad0);
            sad1 = fmaf(sad1c, scale, sad1);
            sad2 = fmaf(sad2c, scale, sad2);
            sad3 = fmaf(sad3c, scale, sad3);
          }
          const float sd[4] = {sad0, sad1, sad2, sad3};
          float w = 1.0f;
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const float wt = epf_weight(sd[k], inv_sigma);
            w = w + wt;
            X = fmaf(wt, nb[0][k], X);
            Y = fmaf(wt, nb[1][k], Y);
            B = fmaf(wt, nb[2][k], B);
          }
          const float inv_w = 1.0f / w;
          X = X * inv_w; Y = Y * inv_w; B = B * inv_w;
        }
        deliver(IC<3>(), r, col, X, Y, B);
      }
    }
    // ---- EPF2 (stage_epf.cc:383-506) ----
    if constexpr (C::E2) {
      const int r = rin - d2;
      const bool row_on = ST || (r >= lo(0) && r < hi(0));
      if (row_on && !(J >= 0 && ((J - d2) & 7) != 0)) load_sel(r, colE2, sgE2, cnE2);
      const int col = colE2;
      const int* cnk = cnE2;
      if (row_on && lane_run(steady_tag, col, h2)) {
        const float s = sgE2;
        const float* pM = RP(ring2, IC<C::N2>(), IC<-d2>(), r);
        float X = pM[col];
        float Y = pM[kStripThreads + col];
        float B = pM[2 * kStripThreads + col];
        if (!(s < kMinSigma)) {
          const int iy = r & 7;
          const float sm_ = P.epf_sm[2];
          const float vsm = (iy == 0 || iy == 7 || xborder) ? sm_ * P.epf_border_mul : sm_;
          const float inv_sigma = s * vsm;
          const float* pT = RP(ring2, IC<C::N2>(), IC<-d2 - 1>(), mr(r - 1));
          const float* pB = RP(ring2, IC<C::N2>(), IC<-d2 + 1>(), mr(r + 1));
          const float* nr[4] = {pT, pM, pM, pB};
          const int nc[4] = {col, EDGE ? cnk[2] : col - 1, EDGE ? cnk[4] : col + 1, col};
          const float rx = X, ry = Y, rb = B;
          float w = 1.0f;
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const float cx = nr[k][nc[k]];
            const float cy = nr[k][kStripThreads + nc[k]];
            const float cb = nr[k][2 * kStripThreads + nc[k]];
            float sad = fabsf(cx - rx) * P.epf_scale[0];
            sad = fmaf(fabsf(cy - ry), P.epf_scale[1], sad);
            sad = fmaf(fabsf(cb - rb), P.epf_scale[2], sad);
            const float wt = epf_weight(sad, inv_sigma);
            w = w + wt;
            X = fmaf(wt, cx, X);
            Y = fmaf(wt, cy, Y);
            B = fmaf(wt, cb, B);
          }
          const float inv_w = 1.0f / w;
          X = X * inv_w; Y = Y * inv_w; B = B * inv_w;
        }
        deliver(IC<4>(), r, col, X, Y, B);
      }
    }
    if constexpr (H > 0) __syncthreads();
  };

  // Steady interval of rin: every stage's row r = rin - d is produced this step (inside its row
  // range) and its whole input window r-b .. r+b lies inside the image (no mirroring).
  int s_lo = r_in_lo, s_hi = r_in_hi;
  auto constrain = [&](int d, int b, int rem) {
    s_lo = max(s_lo, max(lo(rem), b) + d);
    s_hi = min(s_hi, min(hi(rem), HI - b) + d);
  };
  if (C::G) constrain(dG, 1, H - hG);
  if (C::E0) constrain(d0, 3, H - h0);
  if (C::E1) constrain(d1, 2, H - h1);
  if (C::E2) constrain(d2, 1, 0);
  if (s_hi < s_lo) s_hi = s_lo;
  const int s_begin = min(s_lo, r_end), s_end = min(s_hi, r_end);
  using F = std::false_type;
  using T = std::true_type;
  // Fused all-gather: rows this CTA has finished (and that a __syncthreads() made visible) are
  // replayed to the peers every few steps, so the NVLink traffic is spread over the whole kernel.
  constexpr bool replicate = REPL;  // separate instantiation: the single-GPU kernel carries none of this
  const int ncols_out = min(C::kOutCols, W - x0);
  int replayed = y_begin;
  auto replay_to = [&](int row_excl) {
    if constexpr (H == 0) __syncthreads();  // (chains with filters end every step with a barrier)
    row_excl = min(row_excl, y_end);
    for (int y = replayed; y < row_excl; y++) {
      const size_t yo = (size_t)(y - (int)P.out_y0);
      if (P.out_format == 1) {
        for (int c = 0; c < 3; c++)
          replicate_span(P, out, ((size_t)c * band_h + yo) * out_row_stride + (size_t)x0 * 4, ncols_out * 4);
      } else {
        const int pxb = out_pixel_bytes(P.out_format);
        replicate_span(P, out, yo * out_row_stride + (size_t)x0 * pxb, ncols_out * pxb);
      }
    }
    if (row_excl > replayed) replayed = row_excl;
  };
  int rin = r_in_lo;
  for (; rin < s_begin; rin++) step(F(), IC<-1>(), rin);
  if constexpr (H > 0 && !C::E0) {
    // 8x unrolled steady loop with compile-time ring slots (EPF0 chains are too large to replicate)
    if (C::kCompact && rin < s_end) {  // (an unaligned step loads every pass's block selection: the aligned
      step(T(), IC<-1>(), rin);        //  steps below reload it only where a block row begins)
      rin++;
    }
    for (; rin < s_end && (rin & 7); rin++) step(T(), IC<-1>(), rin);
    for (; rin + 8 <= s_end; rin += 8) {
      step(T(), IC<0>(), rin);
      step(T(), IC<1>(), rin + 1);
      step(T(), IC<2>(), rin + 2);
      step(T(), IC<3>(), rin + 3);
      step(T(), IC<4>(), rin + 4);
      step(T(), IC<5>(), rin + 5);
      step(T(), IC<6>(), rin + 6);
      step(T(), IC<7>(), rin + 7);
      if constexpr (replicate) replay_to(rin + 8 - d2);  // rows < rin + 8 - d2 have been emitted
    }
  }
  for (; rin < s_end; rin++) {
    step(T(), IC<-1>(), rin);
    if constexpr (replicate) {
      if ((rin & 7) == 7) replay_to(rin + 1 - d2);
    }
  }
  for (; rin < r_end; rin++) step(F(), IC<-1>(), rin);
  if constexpr (replicate) replay_to(y_end);
}

template <uint32_t MASK, bool REPL, int OUTK>
__global__ void __launch_bounds__(kStripThreads, StripCfg<MASK>::E0 ? 2 : 4) filter_strip_kernel(const __grid_constant__ FrameDev P,
                                                                    char* __restrict__ out,
                                                                    size_t out_row_stride, int seg_rows) {
  extern __shared__ __align__(16) float fsm[];
  using C = StripCfg<MASK>;
  const int x0 = blockIdx.x * C::kOutCols;
  const int y_begin = (int)P.band_y0 + blockIdx.y * seg_rows;
  const int y_end = min((int)P.band_y1, y_begin + seg_rows);
  if (y_begin >= y_end) return;
  const bool edge = (x0 - C::LEAD < 0) || (x0 - C::LEAD + kStripThreads > (int)P.xsize);
  if (edge) filter_strip_body<MASK, true, REPL, OUTK>(P, out, out_row_stride, x0, y_begin, y_end, fsm);
  else filter_strip_body<MASK, false, REPL, OUTK>(P, out, out_row_stride, x0, y_begin, y_end, fsm);
}


// Host launcher of one stage chain; each explicit specialisation lives in its own translation unit
// (jxl_strip_inst.cu compiled with -DSTRIP_MASK=<mask>), so that the eight chains build in parallel.
template <uint32_t MASK>
cudaError_t launch_strip_mask(const FrameDev& P, char* dev_out, size_t out_row_bytes, int num_sms, cudaStream_t s);
// per device, once: opt in to the dynamic shared memory the rings need
template <uint32_t MASK>
__attribute__((visibility("hidden"))) cudaError_t prepare_strip_mask();
#define JXLB_DECLARE_STRIP(M)                                                            \
  template <>                                                                            \
  cudaError_t launch_strip_mask<M>(const FrameDev&, char*, size_t, int, cudaStream_t);   \
  template <>                                                                            \
  __attribute__((visibility("hidden"))) cudaError_t prepare_strip_mask<M>();
JXLB_DECLARE_STRIP(16) JXLB_DECLARE_STRIP(17) JXLB_DECLARE_STRIP(20) JXLB_DECLARE_STRIP(21)
JXLB_DECLARE_STRIP(28) JXLB_DECLARE_STRIP(29) JXLB_DECLARE_STRIP(30) JXLB_DECLARE_STRIP(31)
#undef JXLB_DECLARE_STRIP

// The fused decode kernel (jxl_fused.cuh), one translation unit per stage chain (jxl_fused_inst.cu).
template <uint32_t MASK>
cudaError_t launch_fused_mask(const FrameDev& P, char* dev_out, size_t out_row_bytes, int num_sms, cudaStream_t s);
template <uint32_t MASK>
__attribute__((visibility("hidden"))) cudaError_t prepare_fused_mask();
#define JXLB_DECLARE_FUSED(M)                                                            \
  template <>                                                                            \
  cudaError_t launch_fused_mask<M>(const FrameDev&, char*, size_t, int, cudaStream_t);   \
  template <>                                                                            \
  __attribute__((visibility("hidden"))) cudaError_t prepare_fused_mask<M>();
JXLB_DECLARE_FUSED(16) JXLB_DECLARE_FUSED(17) JXLB_DECLARE_FUSED(20) JXLB_DECLARE_FUSED(21)
JXLB_DECLARE_FUSED(28) JXLB_DECLARE_FUSED(29) JXLB_DECLARE_FUSED(30)
#undef JXLB_DECLARE_FUSED

}  // namespace jxlb
