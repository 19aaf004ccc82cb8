// jxl_b200.cu -- context management and the C ABI of include/jxl_b200.h.
// The product path: there is NO CPU fallback in this library; without a CUDA device every
// entry point fails with JXLGPU_ERR_NO_DEVICE / JXLGPU_ERR_CUDA.
//
// Two ways to run a frame:
//   * device-resident (jxlgpu_set_device_coefficients + jxlgpu_render_device): the whole band in
//     one go on the caller's stream: plan -> IDCT kernels -> filter.
//   * host-fed (jxlgpu_frame_begin / jxlgpu_submit_group / jxlgpu_frame_finish): coefficient
//     groups arrive from the host's worker threads in any order.  As soon as every group of an
//     AC-group row has been submitted, that row's plan+IDCT is enqueued; as soon as rows g-1, g,
//     g+1 are transformed, row g is filtered and -- when the output buffer was announced with
//     jxlgpu_frame_set_output -- copied back.  H2D of later rows, kernels and D2H of earlier rows
//     overlap (three engines: copy-in, SMs, copy-out).
#include "../../include/jxl_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "jxl_kernels.cuh"
#include "jxl_fused.cuh"

using namespace jxlb;

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

}  // namespace

struct jxlgpu_ctx {
  int device = 0;
  uint32_t num_threads = 1;
  cudaStream_t stream = nullptr;                 // compute (and side-info upload) stream
  cudaStream_t s_mid = nullptr, s_large = nullptr, s_down = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_mid = nullptr, ev_large = nullptr, ev_filter = nullptr, ev_ext = nullptr;
  cudaEvent_t ev_ext_done = nullptr;  // last render_device on a caller's stream: the next frame_begin's uploads wait for it
  bool ext_pending = false;
  std::vector<cudaStream_t> up_streams;
  std::vector<cudaEvent_t> up_events;
  // row_events[r]: recorded on the upload stream after the latest copy of AC-group row r, so that
  // a row's kernels wait for exactly that row's DMAs and nothing enqueued later
  std::vector<cudaEvent_t> row_events;
  std::vector<uint8_t> row_event_used;
  uint32_t row_cap = 0;
  int num_sms = 132;   // replaced by the device's count in jxlgpu_create
  bool in_frame = false;
  bool coeff_external = false;
  FrameDev P{};
  uint32_t halo = 0;
  uint32_t num_groups = 0;
  uint32_t need_row0 = 0, need_row1 = 0;         // AC-group rows this band needs (band +- halo)
  uint32_t band_row0 = 0, band_row1 = 0;         // AC-group rows this band renders
  size_t elem_size = 2;
  // streaming state (guarded by mu)
  std::vector<uint8_t> submitted;
  std::vector<uint32_t> row_count;               // groups submitted per group row
  std::vector<size_t> row_bytes;                 // coefficient bytes uploaded per group row
  size_t launch_bytes = 10u << 20;
  uint32_t groups_in = 0;                        // submitted groups among the rows this band needs
  std::vector<uint8_t> row_idct, row_filtered;
  void* host_out = nullptr;
  size_t host_out_stride = 0;
  int stream_error = 0;
  DevBuf acs, quant, sharp, ytox, ytob, dc, dq, coeff, sigma, list, counts, xyb, out;
  DevBuf xyb_rows;            // jxlgpu_device_xyb: row-major copy of the (block-tiled) XYB intermediate
  // multi-GPU gather through the copy engines: finished row chunks are copied to the peers' frame buffers on
  // side streams while the next chunk is filtered (JXLGPU_GATHER=kernel keeps the in-kernel replay)
  cudaStream_t rep_streams[8] = {};
  cudaEvent_t ev_chunk[8] = {}, ev_rep[8] = {};
  bool gather_in_kernel = false;
  bool gather_sm = false;     // JXLGPU_GATHER=sm: peer_copy_kernel per row chunk instead of copy-engine copies
  DevBuf bmap;                // fused path: one 16-byte record per 8x8 block (plan kernel)
  // JXLGPU_FUSED=1 selects the fused decode kernel (jxl_fused.cuh).  Opt-in: it moves 2x fewer DRAM bytes than
  // the two-kernel path but issues about twice the instructions at a third of the occupancy (DESIGN.md §4.8).
  bool allow_fused = false;
  bool idct8_tma = true;      // JXLGPU_IDCT8_TMA=0: the round-1 idct8_kernel (ordinary loads) for A/B runs
  DevBuf ups_in, ups_kern;    // upsampling / noise: filtered XYB planes at the coded size, the N*N x 25 tap table
  DevBuf noise_buf, noise_raw; // noise at the output size: the convolved planes the finish kernels read / the generator's output
  DevBuf qdc, dc_deq;         // DC stage on the device: quantised planes (+ per-group mul), dequantised planes
  DevBuf sparse;              // staging for the non-zero lists of jxlgpu_submit_groups_sparse
  size_t sparse_used = 0;     // words handed out this frame (bump allocation, guarded by mu)
  size_t out_row_bytes = 0;   // dense row of the context-owned output buffer
  std::atomic<uint64_t> launches{0};
  bool force_generic_filter = false;  // JXLGPU_FORCE_GENERIC_FILTER=1: tile kernel for every chain
  bool profile = false;               // record CUDA events around every kernel (bench roofline)
  cudaEvent_t prof_ev[6] = {};
  std::string last_error;
  std::mutex mu;
};

namespace {

int fail_cuda(jxlgpu_ctx* ctx, cudaError_t e, const char* what) {
  ctx->last_error = std::string(what) + ": " + cudaGetErrorString(e);
  return e == cudaErrorMemoryAllocation ? JXLGPU_ERR_OUT_OF_MEMORY : JXLGPU_ERR_CUDA;
}

#define CU(call)                                           \
  do {                                                     \
    cudaError_t e_ = (call);                               \
    if (e_ != cudaSuccess) return fail_cuda(ctx, e_, #call); \
  } while (0)

size_t out_bytes_per_row(const jxlgpu_frame& f) { return (size_t)f.xsize * out_pixel_bytes(f.out_format); }
size_t out_planes(uint32_t out_format) { return out_format == JXLGPU_OUT_PLANAR_F32 ? 3 : 1; }
// alignment the store instructions of a layout need from the row stride (and base pointer)
size_t out_align(uint32_t out_format) {
  switch (out_format) {
    case JXLGPU_OUT_RGB_U8: return 1;
    case JXLGPU_OUT_RGB_U16: case JXLGPU_OUT_RGB_F16: return 2;
    default: return 4;
  }
}

// copies a strided host plane into a dense device plane (one linear DMA when it is dense)
template <typename T>
cudaError_t upload_plane(void* dst, const T* src, size_t stride, size_t w, size_t h, cudaStream_t s) {
  if (stride == w) return cudaMemcpyAsync(dst, src, w * h * sizeof(T), cudaMemcpyHostToDevice, s);
  return cudaMemcpy2DAsync(dst, w * sizeof(T), src, stride * sizeof(T), w * sizeof(T), h,
                           cudaMemcpyHostToDevice, s);
}

// rows of the output buffer -> host (linear DMA when the host rows are dense)
cudaError_t download_rows(void* dst, size_t dst_stride, const void* src, size_t row_bytes, size_t rows,
                          cudaStream_t s) {
  if (dst_stride == row_bytes) return cudaMemcpyAsync(dst, src, row_bytes * rows, cudaMemcpyDeviceToHost, s);
  return cudaMemcpy2DAsync(dst, dst_stride, src, row_bytes, row_bytes, rows, cudaMemcpyDeviceToHost, s);
}

uint32_t effective_mask(const jxlgpu_frame& f) {
  if (f.stage_mask & JXLGPU_STAGE_EXPLICIT) return f.stage_mask & 63u;
  uint32_t m = JXLGPU_STAGE_XYB | (f.stage_mask & JXLGPU_STAGE_SRGB);  // PassesDecoderState::PreparePipeline order, dec_cache.cc:151-170
  if (f.gab) m |= JXLGPU_STAGE_GAB;
  if (f.epf_iters >= 3) m |= JXLGPU_STAGE_EPF0;
  if (f.epf_iters >= 1) m |= JXLGPU_STAGE_EPF1;
  if (f.epf_iters >= 2) m |= JXLGPU_STAGE_EPF2;
  return m;
}

// the stage chains PreparePipeline can build for a VarDCT XYB frame (dec_cache.cc:151-170)
bool launch_strip(jxlgpu_ctx* ctx, const FrameDev& P, char* dev_out, size_t out_row_stride, cudaStream_t s,
                  cudaError_t* err) {
  if (ctx->force_generic_filter) return false;
  switch (P.stage_mask & 31u) {  // (bit 32, the transfer function, is a run-time branch of the store)
    case 16: *err = launch_strip_mask<16>(P, dev_out, out_row_stride, ctx->num_sms, s); return true;
    case 17: *err = launch_strip_mask<17>(P, dev_out, out_row_stride, ctx->num_sms, s); return true;
    case 20: *err = launch_strip_mask<20>(P, dev_out, out_row_stride, ctx->num_sms, s); return true;
    case 21: *err = launch_strip_mask<21>(P, dev_out, out_row_stride, ctx->num_sms, s); return true;
    case 28: *err = launch_strip_mask<28>(P, dev_out, out_row_stride, ctx->num_sms, s); return true;
    case 29: *err = launch_strip_mask<29>(P, dev_out, out_row_stride, ctx->num_sms, s); return true;
    case 30: *err = launch_strip_mask<30>(P, dev_out, out_row_stride, ctx->num_sms, s); return true;
    case 31: *err = launch_strip_mask<31>(P, dev_out, out_row_stride, ctx->num_sms, s); return true;
    default: return false;
  }
}

// The fused decode kernel (jxl_fused.cuh) exists for the chains below; it needs 16-byte aligned coefficient
// planes (bulk copies) and no multicast replica.  (Gaborish + all three EPF passes does not fit its
// shared-memory rings yet and stays on the two-kernel path.)
bool fused_chain(uint32_t mask) {
  switch (mask & 31u) {
    case 16: case 17: case 20: case 21: case 28: case 29: case 30: return true;
    default: return false;
  }
}
// The kernels load whole elements from the coefficient planes: a caller's device-resident planes
// (jxlgpu_set_device_coefficients) must be aligned to the frame's element size.
bool coeff_planes_aligned(jxlgpu_ctx* ctx) {
  for (int c = 0; c < 3; c++)
    if ((uintptr_t)ctx->P.coeff[c] % ctx->elem_size) {
      ctx->last_error = "coefficient planes must be aligned to the element size of the frame's ac_type";
      return false;
    }
  return true;
}

bool use_fused(const jxlgpu_ctx* ctx) {
  const FrameDev& P = ctx->P;
  if (!ctx->allow_fused || ctx->force_generic_filter || !fused_chain(P.stage_mask) || P.mc || P.ups || P.noise || P.ycbcr) return false;
  for (int c = 0; c < 3; c++)
    if ((uintptr_t)P.coeff[c] % 16) return false;
  return true;
}

cudaError_t launch_fused(jxlgpu_ctx* ctx, const FrameDev& P, char* dev_out, size_t out_row_stride, cudaStream_t s) {
  switch (P.stage_mask & 31u) {
    case 16: return launch_fused_mask<16>(P, dev_out, out_row_stride, ctx->num_sms, s);
    case 17: return launch_fused_mask<17>(P, dev_out, out_row_stride, ctx->num_sms, s);
    case 20: return launch_fused_mask<20>(P, dev_out, out_row_stride, ctx->num_sms, s);
    case 21: return launch_fused_mask<21>(P, dev_out, out_row_stride, ctx->num_sms, s);
    case 28: return launch_fused_mask<28>(P, dev_out, out_row_stride, ctx->num_sms, s);
    case 29: return launch_fused_mask<29>(P, dev_out, out_row_stride, ctx->num_sms, s);
    default: return launch_fused_mask<30>(P, dev_out, out_row_stride, ctx->num_sms, s);
  }
}

// plan + inverse transforms of AC-group rows [row0, row1), restricted to the varblocks that
// intersect pixel rows [need_y0, need_y1).  On the fused path only the varblocks larger than 8x8 are
// transformed here (into the XYB planes); the 8x8 class is left to the fused kernel.
int launch_idct(jxlgpu_ctx* ctx, uint32_t row0, uint32_t row1, uint32_t need_y0, uint32_t need_y1, cudaStream_t s) {
  FrameDev P = ctx->P;
  P.plan_g0 = row0 * P.xg;
  P.need_y0 = need_y0;
  P.need_y1 = need_y1;
  const uint32_t plan_groups = (row1 - row0) * P.xg;
  if (!plan_groups) return JXLGPU_OK;
  const bool prof = ctx->profile;
  const bool fused = use_fused(ctx);
  P.fused = fused ? 1u : 0u;
  CU(cudaMemsetAsync(ctx->counts.p, 0, kCountWords * sizeof(uint32_t), s));  // (the 8x8 kernel's work counter too)
  const int want_sigma = (P.stage_mask & 14u) ? 1 : 0;
  if (prof) CU(cudaEventRecord(ctx->prof_ev[0], s));
  plan_kernel<<<plan_groups, 1024, 0, s>>>(P, want_sigma);
  if (prof) CU(cudaEventRecord(ctx->prof_ev[1], s));
  // grids: persistent, never larger than the work (one CTA round = 32 8x8 blocks)
  const uint32_t px_blocks = plan_groups * 1024u;
  int grid8 = ctx->num_sms * 4;  // idct8_kernel: __launch_bounds__(256, 4)
  if ((uint32_t)grid8 > px_blocks / 32u + 1u) grid8 = (int)(px_blocks / 32u + 1u);
  int grid_mid = ctx->num_sms * 2, grid_large = ctx->num_sms * 2;
  if ((uint32_t)grid_mid > px_blocks / 32u + 1u) grid_mid = (int)(px_blocks / 32u + 1u);
  if ((uint32_t)grid_large > px_blocks / 16u + 1u) grid_large = (int)(px_blocks / 16u + 1u);
  // The mid/large kernels usually have little work: run them beside the 8x8 kernel (fork/join)
  // unless per-kernel times are being measured.
  cudaStream_t sm = prof ? s : ctx->s_mid, sl = prof ? s : ctx->s_large;
  if (!prof) {
    CU(cudaEventRecord(ctx->ev_fork, s));
    CU(cudaStreamWaitEvent(sm, ctx->ev_fork, 0));
    CU(cudaStreamWaitEvent(sl, ctx->ev_fork, 0));
  }
  auto run8 = [&]() {
    if (fused) return;  // (the fused kernel transforms the 8x8 class itself)
    bool tma = ctx->idct8_tma;
    for (int c = 0; c < 3; c++) tma = tma && (uintptr_t)P.coeff[c] % 16 == 0;
    if (tma) {  // coefficients staged by the bulk-copy unit one item ahead (2 CTAs of 16 warps per SM)
      int grid = ctx->num_sms * 2;
      if ((uint32_t)grid > px_blocks / 64u + 1u) grid = (int)(px_blocks / 64u + 1u);  // 64 blocks per CTA round
      if (P.ac_is32) idct8_tma_kernel<true><<<grid, kTma8Warps * 32, kTma8SmemBytes, s>>>(P);
      else idct8_tma_kernel<false><<<grid, kTma8Warps * 32, kTma8SmemBytes, s>>>(P);
      return;
    }
    if (P.ac_is32) idct8_kernel<true><<<grid8, kSmallWarpsPerCta * 32, 0, s>>>(P);
    else idct8_kernel<false><<<grid8, kSmallWarpsPerCta * 32, 0, s>>>(P);
  };
  if (prof) {
    run8();
    CU(cudaEventRecord(ctx->prof_ev[2], s));
  }
  if (P.ac_is32) idct_mid_kernel<true><<<grid_mid, kSmallWarpsPerCta * 32, 0, sm>>>(P);
  else idct_mid_kernel<false><<<grid_mid, kSmallWarpsPerCta * 32, 0, sm>>>(P);
  if (prof) CU(cudaEventRecord(ctx->prof_ev[3], s));
  // two launches: row slabs, then column slabs (jxl_kernels.cuh: large_item)
  constexpr size_t kLargeSmem = kLargeSmemFloats * sizeof(float);
  if (P.ac_is32) {
    idct_large_kernel<true, 0><<<grid_large, kLargeWarps * 32, kLargeSmem, sl>>>(P);
    idct_large_kernel<true, 1><<<grid_large, kLargeWarps * 32, kLargeSmem, sl>>>(P);
  } else {
    idct_large_kernel<false, 0><<<grid_large, kLargeWarps * 32, kLargeSmem, sl>>>(P);
    idct_large_kernel<false, 1><<<grid_large, kLargeWarps * 32, kLargeSmem, sl>>>(P);
  }
  if (prof) CU(cudaEventRecord(ctx->prof_ev[4], s));
  // The side kernels go first: launched after it, they would find every SM full of 8x8 CTAs and start only as
  // those finish (where they have real work, e.g. all-27-strategy frames, they are the longer chain).  While one of
  // their CTAs is resident (mid: 126 registers x 256 threads, large: 107 KB of shared memory), its SM holds one 8x8
  // CTA instead of two; the 8x8 kernel's warps claim their items from a counter, so the CTAs that start late just
  // do fewer (DESIGN.md §4, item 2).
  if (!prof) run8();
  if (!prof) {
    CU(cudaEventRecord(ctx->ev_mid, sm));
    CU(cudaEventRecord(ctx->ev_large, sl));
    CU(cudaStreamWaitEvent(s, ctx->ev_mid, 0));
    CU(cudaStreamWaitEvent(s, ctx->ev_large, 0));
  }
  ctx->launches += fused ? 4 : 5;
  CU(cudaGetLastError());
  return JXLGPU_OK;
}

// filters pixel rows [y0, y1) into dev_out, whose row 0 is image row out_y0.
int launch_filter(jxlgpu_ctx* ctx, uint32_t y0, uint32_t y1, uint32_t out_y0, uint32_t out_h, char* dev_out,
                  size_t out_row_stride, cudaStream_t s) {
  if (y1 <= y0) return JXLGPU_OK;
  FrameDev P = ctx->P;
  P.band_y0 = y0;
  P.band_y1 = y1;
  P.out_y0 = out_y0;
  P.out_h = out_h;
  if (P.ups || P.noise) {
    // the filters run at the coded size into planar XYB; upsample_kernel (launch_upsample) carries the
    // stages behind the upsampling: XYB -> RGB, transfer function, packing
    // (the production chains keep their strip-kernel instantiation: the XYB bit stays in the mask, the kernel
    //  skips the conversion at run time; other chains run the generic tile kernel without the bit)
    const bool strip_chain = !ctx->force_generic_filter && (P.stage_mask & 16u);
    P.skip_xyb = strip_chain ? 1u : 0u;
    P.stage_mask &= strip_chain ? 31u : 15u;
    P.out_format = 1;
    P.out_y0 = 0;
    P.out_h = P.ysize;
    P.nrep = 0;
    P.mc = nullptr;
    dev_out = (char*)ctx->ups_in.p;
    out_row_stride = (size_t)P.xsize * 4;
  }
  cudaError_t strip_err = cudaSuccess;
  if (!(P.ups || P.noise) && use_fused(ctx)) {
    // coefficients -> pixels in one kernel; finished rows leave through the TMA unit when every row
    // segment is 16-byte aligned (the kernel checks the per-strip size)
    bool aligned = (uintptr_t)dev_out % 16 == 0 && out_row_stride % 16 == 0;
    for (uint32_t q = 0; q < P.nrep; q++) aligned = aligned && (uintptr_t)P.rep[q] % 16 == 0;
    P.fused = 1u | (aligned ? 2u : 0u);
    strip_err = launch_fused(ctx, P, dev_out, out_row_stride, s);
  } else if (!launch_strip(ctx, P, dev_out, out_row_stride, s, &strip_err)) {
    // stage chains outside the production set (test taps): generic tile kernel.  It has no skip_xyb: in front
    // of the upsampling its mask must stop before XYB -> RGB (an explicit chain keeps the bit up to here)
    if (P.skip_xyb) {
      P.stage_mask &= 15u;
      P.skip_xyb = 0;
    }
    dim3 grid((P.xsize + kTW - 1) / kTW, (y1 - y0 + kTH - 1) / kTH);
    filter_kernel<<<grid, kFilterThreads, kFilterSmemFloats * sizeof(float), s>>>(P, dev_out, out_row_stride);
  }
  CU(strip_err);
  if (ctx->profile) CU(cudaEventRecord(ctx->prof_ev[5], s));
  ctx->launches += 1;
  CU(cudaGetLastError());
  return JXLGPU_OK;
}

// the whole frame: filtered planes (ups_in) -> upsampled, colour-converted, packed pixels
int launch_upsample(jxlgpu_ctx* ctx, char* dev_out, size_t out_row_stride, cudaStream_t s) {
  FrameDev P = ctx->P;
  P.out_y0 = 0;
  P.out_h = P.out_hh;
  const float* src = (const float*)ctx->ups_in.p;
  if (P.ups) {  // one thread per input pixel (window loaded once for its N x N outputs)
    const dim3 gi((P.xsize + 31) / 32, (P.ysize + 7) / 8);
    if (P.ups == 2) upsample_in_kernel<2><<<gi, 256, 0, s>>>(P, src, dev_out, out_row_stride);
    else if (P.ups == 4) upsample_in_kernel<4><<<gi, 256, 0, s>>>(P, src, dev_out, out_row_stride);
    else upsample_in_kernel<8><<<gi, 256, 0, s>>>(P, src, dev_out, out_row_stride);
  } else {      // noise only: one thread per output (= input) pixel
    const dim3 grid((P.out_w + 31) / 32, (P.out_hh + 7) / 8);
    upsample_kernel<<<grid, 256, 0, s>>>(P, src, dev_out, out_row_stride);
  }
  ctx->launches += 1;
  CU(cudaGetLastError());
  return JXLGPU_OK;
}

int ensure_out(jxlgpu_ctx* ctx) {
  const uint32_t band_h = (ctx->P.ups || ctx->P.noise) ? ctx->P.out_hh : ctx->P.band_y1 - ctx->P.band_y0;
  CU(ctx->out.ensure(out_planes(ctx->P.out_format) * band_h * ctx->out_row_bytes));
  return JXLGPU_OK;
}

// Streaming scheduler, called with ctx->mu held: enqueue whatever became runnable.
// Granularity: kernels are launched over runs of complete AC-group rows.  A run is launched once
// the coefficient bytes uploaded for it amount to kLaunchBytes (~0.2 ms of PCIe time: with dense 8K
// rows that is every row, with sparse lists every ~3 rows; measured best of 3/8/20 MB), when
// the band's last group has arrived, or when frame_finish forces it -- so a PCIe-bound feed keeps
// its per-row overlap and a light feed does not pay 17 under-filled launches per frame.
constexpr size_t kLaunchBytes = 10u << 20;  // (JXLGPU_LAUNCH_MB overrides it: tuning knob)

int pump(jxlgpu_ctx* ctx, bool force) {
  const FrameDev& P = ctx->P;
  cudaStream_t s = ctx->stream;
  if (ctx->coeff_external || ctx->groups_in == (ctx->need_row1 - ctx->need_row0) * P.xg) force = true;
  for (uint32_t g = ctx->need_row0; g < ctx->need_row1;) {
    if (ctx->row_idct[g] || ctx->row_count[g] < P.xg) {
      g++;
      continue;
    }
    uint32_t h = g;
    size_t bytes = 0;
    while (h < ctx->need_row1 && !ctx->row_idct[h] && ctx->row_count[h] == P.xg) bytes += ctx->row_bytes[h++];
    if (!force && bytes < ctx->launch_bytes) {
      g = h;
      continue;
    }
    // the rows' coefficients are in flight on the upload stream
    if (!ctx->coeff_external)
      for (uint32_t r = g; r < h; r++)
        if (ctx->row_event_used[r]) CU(cudaStreamWaitEvent(s, ctx->row_events[r], 0));
    uint32_t ny0 = g * 256u, ny1 = h * 256u;
    if (ny0 < P.need_y0) ny0 = P.need_y0;
    if (ny1 > P.need_y1 || h == ctx->need_row1) ny1 = P.need_y1;
    int rc = launch_idct(ctx, g, h, ny0, ny1, s);
    if (rc) return rc;
    for (uint32_t r = g; r < h; r++) ctx->row_idct[r] = 1;
    g = h;
  }
  // filter every run of rows whose neighbours (the 7-row halo) are transformed
  const uint32_t band_h = P.band_y1 - P.band_y0;
  auto ready = [&](uint32_t g) {
    if (ctx->row_filtered[g]) return false;
    const uint32_t lo = g > ctx->need_row0 ? g - 1 : g;
    const uint32_t hi = g + 1 < ctx->need_row1 ? g + 1 : g;
    for (uint32_t r = lo; r <= hi; r++)
      if (!ctx->row_idct[r]) return false;
    return true;
  };
  for (uint32_t g = ctx->band_row0; g < ctx->band_row1;) {
    if (!ready(g)) {
      g++;
      continue;
    }
    uint32_t h = g + 1;
    while (h < ctx->band_row1 && ready(h)) h++;
    uint32_t y0 = g * 256u, y1 = h * 256u;
    if (y0 < P.band_y0) y0 = P.band_y0;
    if (y1 > P.band_y1) y1 = P.band_y1;
    int rc = ensure_out(ctx);
    if (rc) return rc;
    rc = launch_filter(ctx, y0, y1, P.band_y0, band_h, (char*)ctx->out.p, ctx->out_row_bytes, s);
    if (rc) return rc;
    for (uint32_t r = g; r < h; r++) ctx->row_filtered[r] = 1;
    if (ctx->host_out && y1 > y0 && !(P.ups || P.noise)) {  // copy the finished rows back while later rows still arrive
      CU(cudaEventRecord(ctx->ev_filter, s));
      CU(cudaStreamWaitEvent(ctx->s_down, ctx->ev_filter, 0));
      const size_t row_bytes = ctx->out_row_bytes;
      const size_t planes = out_planes(P.out_format);
      for (size_t pl = 0; pl < planes; pl++) {
        const size_t row = pl * band_h + (y0 - P.band_y0);
        CU(download_rows((uint8_t*)ctx->host_out + row * ctx->host_out_stride, ctx->host_out_stride,
                         (uint8_t*)ctx->out.p + row * row_bytes, row_bytes, y1 - y0, ctx->s_down));
      }
    }
    g = h;
  }
  return JXLGPU_OK;
}

}  // namespace

extern "C" {

uint32_t jxlgpu_abi_version(void) { return JXLGPU_ABI_VERSION; }

const char* jxlgpu_error_string(int code) {
  switch (code) {
    case JXLGPU_OK: return "ok";
    case JXLGPU_ERR_INVALID_ARGUMENT: return "invalid argument";
    case JXLGPU_ERR_UNSUPPORTED: return "frame not eligible for the GPU path";
    case JXLGPU_ERR_NO_DEVICE: return "no CUDA device";
    case JXLGPU_ERR_CUDA: return "CUDA error";
    case JXLGPU_ERR_OUT_OF_MEMORY: return "out of device memory";
    case JXLGPU_ERR_STATE: return "call out of order";
  }
  return "unknown";
}

const char* jxlgpu_last_error(const jxlgpu_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }

int jxlgpu_create(jxlgpu_ctx** out, const jxlgpu_config* cfg) {
  if (!out || !cfg || cfg->abi_version != JXLGPU_ABI_VERSION) return JXLGPU_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0 || cfg->device < 0 || cfg->device >= n) return JXLGPU_ERR_NO_DEVICE;
  jxlgpu_ctx* ctx = new jxlgpu_ctx();
  ctx->device = cfg->device;
  ctx->num_threads = cfg->num_host_threads ? cfg->num_host_threads : 1;
  auto bail = [&](cudaError_t err, const char* what) {
    fprintf(stderr, "jxlgpu_create: %s: %s\n", what, cudaGetErrorString(err));
    jxlgpu_destroy(ctx);  // releases the streams / events / buffers created so far
    return JXLGPU_ERR_CUDA;
  };
  if ((e = cudaSetDevice(ctx->device)) != cudaSuccess) return bail(e, "cudaSetDevice");
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, ctx->device)) != cudaSuccess) return bail(e, "props");
  ctx->num_sms = prop.multiProcessorCount;
  for (cudaStream_t* sp : {&ctx->stream, &ctx->s_mid, &ctx->s_large, &ctx->s_down})
    if ((e = cudaStreamCreateWithFlags(sp, cudaStreamNonBlocking)) != cudaSuccess) return bail(e, "stream");
  for (cudaEvent_t* ep : {&ctx->ev_fork, &ctx->ev_mid, &ctx->ev_large, &ctx->ev_filter, &ctx->ev_ext, &ctx->ev_ext_done})
    if ((e = cudaEventCreateWithFlags(ep, cudaEventDisableTiming)) != cudaSuccess) return bail(e, "event");
  ctx->up_streams.resize(ctx->num_threads);
  ctx->up_events.resize(ctx->num_threads);
  for (uint32_t i = 0; i < ctx->num_threads; i++) {
    if ((e = cudaStreamCreateWithFlags(&ctx->up_streams[i], cudaStreamNonBlocking)) != cudaSuccess) return bail(e, "stream");
    if ((e = cudaEventCreateWithFlags(&ctx->up_events[i], cudaEventDisableTiming)) != cudaSuccess) return bail(e, "event");
  }
  if ((e = cudaFuncSetAttribute(filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)(kFilterSmemFloats * sizeof(float)))) != cudaSuccess)
    return bail(e, "cudaFuncSetAttribute(filter_kernel)");
  for (cudaError_t ea : {cudaFuncSetAttribute(idct8_tma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTma8SmemBytes),
                         cudaFuncSetAttribute(idct8_tma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTma8SmemBytes)})
    if (ea != cudaSuccess) return bail(ea, "cudaFuncSetAttribute(idct8_tma_kernel)");
  for (cudaError_t ea : {cudaFuncSetAttribute(idct_large_kernel<true, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kLargeSmemFloats * sizeof(float))),
                         cudaFuncSetAttribute(idct_large_kernel<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kLargeSmemFloats * sizeof(float))),
                         cudaFuncSetAttribute(idct_large_kernel<false, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kLargeSmemFloats * sizeof(float))),
                         cudaFuncSetAttribute(idct_large_kernel<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kLargeSmemFloats * sizeof(float)))})
    if (ea != cudaSuccess) return bail(ea, "cudaFuncSetAttribute(idct_large_kernel)");
  for (cudaError_t ea : {prepare_strip_mask<16>(), prepare_strip_mask<17>(), prepare_strip_mask<20>(),
                         prepare_strip_mask<21>(), prepare_strip_mask<28>(), prepare_strip_mask<29>(),
                         prepare_strip_mask<30>(), prepare_strip_mask<31>()})
    if (ea != cudaSuccess) return bail(ea, "cudaFuncSetAttribute(filter_strip_kernel)");
  for (cudaError_t ea : {prepare_fused_mask<16>(), prepare_fused_mask<17>(), prepare_fused_mask<20>(),
                         prepare_fused_mask<21>(), prepare_fused_mask<28>(), prepare_fused_mask<29>(),
                         prepare_fused_mask<30>()})
    if (ea != cudaSuccess) return bail(ea, "cudaFuncSetAttribute(fused_tile_kernel)");
  if (const char* fe = getenv("JXLGPU_FUSED")) ctx->allow_fused = fe[0] == '1';
  if (const char* te = getenv("JXLGPU_IDCT8_TMA")) ctx->idct8_tma = te[0] != '0';
  if (const char* ge = getenv("JXLGPU_GATHER")) {
    ctx->gather_in_kernel = ge[0] == 'k';
    ctx->gather_sm = ge[0] == 's';
  }
  {
    const char* env = getenv("JXLGPU_FORCE_GENERIC_FILTER");
    ctx->force_generic_filter = env && env[0] == '1';
    ctx->launch_bytes = kLaunchBytes;
    if (const char* mb = getenv("JXLGPU_LAUNCH_MB")) ctx->launch_bytes = (size_t)atoi(mb) << 20;
  }
  if ((e = ctx->counts.ensure(kCountWords * sizeof(uint32_t))) != cudaSuccess) return bail(e, "alloc");
  for (auto& ev : ctx->prof_ev)
    if ((e = cudaEventCreate(&ev)) != cudaSuccess) return bail(e, "event");
  *out = ctx;
  return JXLGPU_OK;
}

void jxlgpu_destroy(jxlgpu_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (DevBuf* b : {&ctx->acs, &ctx->quant, &ctx->sharp, &ctx->ytox, &ctx->ytob, &ctx->dc, &ctx->dq,
                    &ctx->coeff, &ctx->sigma,
                    &ctx->list, &ctx->counts, &ctx->xyb, &ctx->xyb_rows, &ctx->out, &ctx->sparse, &ctx->qdc, &ctx->dc_deq, &ctx->bmap})
    b->release();
  for (auto s : ctx->up_streams)
    if (s) cudaStreamDestroy(s);
  for (auto ev : ctx->up_events)
    if (ev) cudaEventDestroy(ev);
  for (auto ev : ctx->row_events)
    if (ev) cudaEventDestroy(ev);
  for (auto ev : ctx->prof_ev)
    if (ev) cudaEventDestroy(ev);
  for (cudaEvent_t ev : {ctx->ev_fork, ctx->ev_mid, ctx->ev_large, ctx->ev_filter, ctx->ev_ext, ctx->ev_ext_done})
    if (ev) cudaEventDestroy(ev);
  for (cudaStream_t s : {ctx->stream, ctx->s_mid, ctx->s_large, ctx->s_down})
    if (s) cudaStreamDestroy(s);
  for (int i = 0; i < 8; i++) {
    if (ctx->rep_streams[i]) cudaStreamDestroy(ctx->rep_streams[i]);
    if (ctx->ev_chunk[i]) cudaEventDestroy(ctx->ev_chunk[i]);
    if (ctx->ev_rep[i]) cudaEventDestroy(ctx->ev_rep[i]);
  }
  delete ctx;
}

int jxlgpu_frame_begin(jxlgpu_ctx* ctx, const jxlgpu_frame* f) {
  if (!ctx || !f) return JXLGPU_ERR_INVALID_ARGUMENT;
  CU(cudaSetDevice(ctx->device));
  if (f->xsize == 0 || f->ysize == 0 || f->xsize_blocks != (f->xsize + 7) / 8 ||
      f->ysize_blocks != (f->ysize + 7) / 8 || f->xsize_blocks > 65535 || f->ysize_blocks > 65535)
    return JXLGPU_ERR_INVALID_ARGUMENT;
  const bool dc_on_device = f->quant_dc[0] != nullptr;
  if (!f->ac_strategy || !f->raw_quant || !f->ytox_map || !f->ytob_map || !f->dequant_table)
    return JXLGPU_ERR_INVALID_ARGUMENT;
  if (dc_on_device ? (!f->quant_dc[1] || !f->quant_dc[2] || f->quant_dc_stride < f->xsize_blocks)
                   : (!f->dc[0] || !f->dc[1] || !f->dc[2]))
    return JXLGPU_ERR_INVALID_ARGUMENT;
  if (f->ac_type > JXLGPU_AC_INT32 || f->out_format > JXLGPU_OUT_RGB_F16) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (f->color_transform > 1) return JXLGPU_ERR_INVALID_ARGUMENT;
  const uint32_t ups = f->upsampling <= 1 ? 0 : f->upsampling;
  uint32_t out_w = f->xsize, out_hh = f->ysize;
  if (ups) {
    if (ups != 2 && ups != 4 && ups != 8) return JXLGPU_ERR_INVALID_ARGUMENT;
    if (!f->upsampling_weights) return JXLGPU_ERR_INVALID_ARGUMENT;
    if (f->band_ny_groups) return JXLGPU_ERR_UNSUPPORTED;  // whole-frame contexts only
    out_w = f->xsize_upsampled ? f->xsize_upsampled : ups * f->xsize;
    out_hh = f->ysize_upsampled ? f->ysize_upsampled : ups * f->ysize;
    // FrameDimensions: size = DivCeil(size_upsampled, upsampling)
    if ((out_w + ups - 1) / ups != f->xsize || (out_hh + ups - 1) / ups != f->ysize) return JXLGPU_ERR_INVALID_ARGUMENT;
  }
  // plane strides (in elements) must cover a row: a short stride would make the uploads read out of bounds
  if (f->ac_strategy_stride < f->xsize_blocks || f->raw_quant_stride < f->xsize_blocks ||
      (f->epf_sharpness && f->epf_sharpness_stride < f->xsize_blocks) ||
      (!dc_on_device && f->dc_stride < f->xsize_blocks) || f->cmap_stride < (f->xsize_blocks + 7) / 8)
    return JXLGPU_ERR_INVALID_ARGUMENT;
  const uint32_t mask = effective_mask(*f);
  if ((mask & 14u) && !f->epf_sharpness) return JXLGPU_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < 3 * kNumStrategies; i++) {
    const size_t n = (size_t)64 * covered_x(i / 3) * covered_y(i / 3);
    if (f->dequant_offsets[i] + n > f->dequant_table_floats) return JXLGPU_ERR_INVALID_ARGUMENT;
    if (f->dequant_offsets[i] % 4) return JXLGPU_ERR_INVALID_ARGUMENT;  // 16-byte vector loads
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  FrameDev& P = ctx->P;
  const size_t xb = f->xsize_blocks, yb = f->ysize_blocks, nblocks = xb * yb;
  P.xsize = f->xsize; P.ysize = f->ysize; P.xb = xb; P.yb = yb;
  P.xg = (xb + 31) / 32; P.yg = (yb + 31) / 32;
  ctx->num_groups = P.xg * P.yg;
  P.ac_is32 = f->ac_type == JXLGPU_AC_INT32;
  ctx->elem_size = P.ac_is32 ? 4 : 2;
  P.stage_mask = mask;
  P.out_format = f->out_format;
  if (f->band_ny_groups == 0) {
    P.band_y0 = 0; P.band_y1 = f->ysize;
    ctx->band_row0 = 0; ctx->band_row1 = P.yg;
  } else {
    if (f->band_y0_groups + f->band_ny_groups > P.yg) return JXLGPU_ERR_INVALID_ARGUMENT;
    P.band_y0 = f->band_y0_groups * 256u;
    const uint32_t y1 = (f->band_y0_groups + f->band_ny_groups) * 256u;
    P.band_y1 = y1 < f->ysize ? y1 : f->ysize;
    ctx->band_row0 = f->band_y0_groups; ctx->band_row1 = f->band_y0_groups + f->band_ny_groups;
  }
  P.out_y0 = P.band_y0;
  P.out_h = P.band_y1 - P.band_y0;
  {
    const uint32_t halo = ((mask & 1) ? 1 : 0) + ((mask & 2) ? 3 : 0) + ((mask & 4) ? 2 : 0) + ((mask & 8) ? 1 : 0);
    ctx->halo = halo;
    P.need_y0 = P.band_y0 > halo ? P.band_y0 - halo : 0;
    P.need_y1 = P.band_y1 + halo < f->ysize ? P.band_y1 + halo : f->ysize;
    if (P.band_y1 >= f->ysize) P.need_y1 = (uint32_t)yb * 8;  // bottom band also owns the padded block rows
    ctx->need_row0 = P.need_y0 / 256;
    const uint32_t gy1 = (P.need_y1 + 255) / 256;
    ctx->need_row1 = gy1 < P.yg ? gy1 : P.yg;
    P.plan_g0 = ctx->need_row0 * P.xg;
  }
  const size_t cmw = (xb + 7) / 8, cmh = (yb + 7) / 8;
  CU(ctx->acs.ensure(nblocks));
  CU(ctx->quant.ensure(nblocks * 4));
  CU(ctx->sharp.ensure(nblocks));
  CU(ctx->ytox.ensure(cmw * cmh));
  CU(ctx->ytob.ensure(cmw * cmh));
  CU(ctx->dc.ensure(3 * nblocks * 4));
  CU(ctx->dq.ensure(f->dequant_table_floats * 4));
  CU(ctx->sigma.ensure(nblocks * 4));
  CU(ctx->bmap.ensure(nblocks * sizeof(uint4)));
  // per-strategy work lists, capacity = max number of varblocks of that size
  size_t total = 0;
  for (int s = 0; s < kNumStrategies; s++) {
    P.list_base[s] = (uint32_t)total;
    total += nblocks / (covered_x(s) * covered_y(s)) + 1;
  }
  CU(ctx->list.ensure(total * sizeof(uint4)));
  P.plane_stride = (size_t)xb * yb * 64;   // [3][yb][xb][64]: 8x8 block tiles (FrameDev::xyb_off)
  CU(ctx->xyb.ensure(3 * P.plane_stride * 4));
  // host-fed coefficients live group-major on the device: [group][channel][65536]
  if (!ctx->coeff_external) CU(ctx->coeff.ensure((size_t)ctx->num_groups * 3 * 65536 * ctx->elem_size));
  cudaStream_t s = ctx->stream;
  if (ctx->ext_pending) {  // kernels of the previous frame may still read the side information on the caller's stream
    CU(cudaStreamWaitEvent(s, ctx->ev_ext_done, 0));
    ctx->ext_pending = false;
  }
  CU(upload_plane<uint8_t>(ctx->acs.p, f->ac_strategy, f->ac_strategy_stride, xb, yb, s));
  CU(upload_plane<int32_t>(ctx->quant.p, f->raw_quant, f->raw_quant_stride, xb, yb, s));
  if (f->epf_sharpness) CU(upload_plane<uint8_t>(ctx->sharp.p, f->epf_sharpness, f->epf_sharpness_stride, xb, yb, s));
  CU(upload_plane<int8_t>(ctx->ytox.p, f->ytox_map, f->cmap_stride, cmw, cmh, s));
  CU(upload_plane<int8_t>(ctx->ytob.p, f->ytob_map, f->cmap_stride, cmw, cmh, s));
  if (!dc_on_device) {
    for (int c = 0; c < 3; c++)
      CU(upload_plane<float>((float*)ctx->dc.p + c * nblocks, f->dc[c], f->dc_stride, xb, yb, s));
  } else {
    // DC stage on the device: quantised planes up, dequantise, smooth (two small launches)
    const uint32_t xdg = (uint32_t)((xb + 255) / 256), ydg = (uint32_t)((yb + 255) / 256);
    CU(ctx->qdc.ensure(3 * nblocks * 4 + (size_t)xdg * ydg * 4));
    CU(ctx->dc_deq.ensure(3 * nblocks * 4));
    DcStage S{};
    S.xb = (uint32_t)xb;
    S.yb = (uint32_t)yb;
    S.xdg = xdg;
    for (int c = 0; c < 3; c++) {
      CU(upload_plane<int32_t>((int32_t*)ctx->qdc.p + c * nblocks, f->quant_dc[c], f->quant_dc_stride, xb, yb, s));
      S.q[c] = (const int32_t*)ctx->qdc.p + c * nblocks;
      S.deq[c] = (float*)ctx->dc_deq.p + c * nblocks;
      S.out[c] = (float*)ctx->dc.p + c * nblocks;
      S.dc_factors[c] = f->dc_factors[c];
    }
    S.cfl_x = f->dc_cfl_factors[0];
    S.cfl_b = f->dc_cfl_factors[2];
    if (f->dc_group_mul) {
      float* gm = (float*)((int32_t*)ctx->qdc.p + 3 * nblocks);
      CU(cudaMemcpyAsync(gm, f->dc_group_mul, (size_t)xdg * ydg * 4, cudaMemcpyHostToDevice, s));
      S.group_mul = gm;
    }
    const dim3 grid((unsigned)((xb + 31) / 32), (unsigned)((yb + 7) / 8));
    dc_dequant_kernel<<<grid, 256, 0, s>>>(S);
    dc_smooth_kernel<<<grid, 256, 0, s>>>(S, f->dc_smoothing ? 1 : 0);
    CU(cudaGetLastError());
    ctx->launches += 2;
  }
  CU(cudaMemcpyAsync(ctx->dq.p, f->dequant_table, f->dequant_table_floats * 4, cudaMemcpyHostToDevice, s));
  P.acs = (const uint8_t*)ctx->acs.p;
  P.quant = (const int32_t*)ctx->quant.p;
  P.sharp = (const uint8_t*)ctx->sharp.p;
  P.ytox = (const int8_t*)ctx->ytox.p;
  P.ytob = (const int8_t*)ctx->ytob.p;
  P.cmap_stride = cmw;
  P.dc = (const float*)ctx->dc.p;
  P.dq = (const float*)ctx->dq.p;
  memcpy(P.dq_off, f->dequant_offsets, sizeof(P.dq_off));
  if (!ctx->coeff_external) {
    for (int c = 0; c < 3; c++) P.coeff[c] = (uint8_t*)ctx->coeff.p + (size_t)c * 65536 * ctx->elem_size;
    P.coeff_gstride = 3 * 65536;
  }
  P.sigma = (float*)ctx->sigma.p;
  P.bmap = (uint4*)ctx->bmap.p;
  P.fused = 0;
  P.skip_xyb = 0;
  P.ycbcr = f->color_transform == 1 ? 1u : 0u;
  P.list = (uint4*)ctx->list.p;
  P.counts = (uint32_t*)ctx->counts.p;
  P.xyb = (float*)ctx->xyb.p;
  P.inv_global_scale = f->inv_global_scale;
  P.quant_scale = f->quant_scale;
  P.x_dm = f->x_dm_multiplier;
  P.b_dm = f->b_dm_multiplier;
  memcpy(P.qbias, f->quant_biases, sizeof(P.qbias));
  P.cfl_base_x = f->cfl_base_x; P.cfl_base_b = f->cfl_base_b; P.cfl_scale = f->cfl_color_scale;
  for (int c = 0; c < 3; c++) {  // GaborishStage ctor (stage_gaborish.cc:33-54)
    float w0 = 1.0f, w1 = f->gab_weights[2 * c], w2 = f->gab_weights[2 * c + 1];
    const float div = w0 + 4 * (w1 + w2);
    const float mul = 1.0f / div;
    P.gab_w[3 * c] = w0 * mul; P.gab_w[3 * c + 1] = w1 * mul; P.gab_w[3 * c + 2] = w2 * mul;
  }
  memcpy(P.epf_sharp_lut, f->epf_sharp_lut, sizeof(P.epf_sharp_lut));
  memcpy(P.epf_scale, f->epf_channel_scale, sizeof(P.epf_scale));
  P.epf_quant_mul = f->epf_quant_mul;
  P.epf_sm[0] = (float)(f->epf_pass0_sigma_scale * 1.65);  // stage_epf.cc:93
  P.epf_sm[1] = 1.65f;                                      // stage_epf.cc:236
  P.epf_sm[2] = (float)(f->epf_pass2_sigma_scale * 1.65);  // stage_epf.cc:427
  P.epf_border_mul = f->epf_border_sad_mul;
  memcpy(P.opsin_m, f->inverse_opsin_matrix, sizeof(P.opsin_m));
  memcpy(P.opsin_bias, f->opsin_biases, sizeof(P.opsin_bias));
  memcpy(P.opsin_cbrt, f->opsin_biases_cbrt, sizeof(P.opsin_cbrt));
  ctx->out_row_bytes = (size_t)out_w * out_pixel_bytes(f->out_format);
  P.ups = ups;
  P.out_w = out_w;
  P.out_hh = out_hh;
  P.ups_kernel = nullptr;
  P.noise = f->noise ? 1u : 0u;
  P.noise_planes = nullptr;
  if (P.noise) {
    if (f->band_ny_groups) return JXLGPU_ERR_UNSUPPORTED;  // whole-frame contexts only
    memcpy(P.noise_lut, f->noise_lut, sizeof(P.noise_lut));
    CU(ctx->noise_buf.ensure((size_t)3 * out_w * out_hh * 4));
    CU(ctx->noise_raw.ensure((size_t)3 * out_w * out_hh * 4));
    CU(ctx->ups_in.ensure((size_t)3 * f->xsize * f->ysize * 4));
    P.noise_planes = (const float*)ctx->noise_buf.p;
    // the planes depend on the frame indices and the output size only: generated while the side information uploads
    const uint32_t tiles = ((out_w + 255) / 256) * ((out_hh + 255) / 256);
    float* const nraw = (float*)ctx->noise_raw.p;
    float* const nconv = (float*)ctx->noise_buf.p;
    noise_gen_kernel<<<(tiles + 3) / 4, 32, 0, s>>>(nraw, out_w, out_hh, f->visible_frame_index, f->nonvisible_frame_index);
    const dim3 cgrid((out_w + 31) / 32, (out_hh + 7) / 8, 3);
    noise_conv_kernel<<<cgrid, 256, 0, s>>>(nraw, nconv, (int)out_w, (int)out_hh);
    CU(cudaGetLastError());
    ctx->launches += 2;
  }
  if (ups) {
    // the stage's constructor (stage_upsampling.cc:61-86): N/2 x N/2 x 25 symmetric weights -> N*N kernels of 25 taps
    const uint32_t N = ups, H = N / 2;
    std::vector<float> kern((size_t)N * N * 25);
    const float* w = f->upsampling_weights;
    for (uint32_t ky = 0; ky < H; ky++)
      for (uint32_t kx = 0; kx < H; kx++) {
        const size_t o0 = (ky * N + kx) * 25, o1 = (ky * N + (N - 1 - kx)) * 25;
        const size_t o2 = ((N - 1 - ky) * N + kx) * 25, o3 = ((N - 1 - ky) * N + (N - 1 - kx)) * 25;
        for (uint32_t py = 0; py < 5; py++)
          for (uint32_t px = 0; px < 5; px++) {
            const uint32_t j = 5 * ky + py, i = 5 * kx + px;
            const uint32_t my = i < j ? i : j, mx = i < j ? j : i;
            const float v = w[5 * H * my - my * (my - 1) / 2 + mx - my];
            kern[o0 + py * 5 + px] = v;
            kern[o1 + py * 5 + (4 - px)] = v;
            kern[o2 + (4 - py) * 5 + px] = v;
            kern[o3 + (4 - py) * 5 + (4 - px)] = v;
          }
      }
    CU(ctx->ups_kern.ensure(kern.size() * 4));
    CU(cudaMemcpyAsync(ctx->ups_kern.p, kern.data(), kern.size() * 4, cudaMemcpyHostToDevice, s));
    CU(cudaStreamSynchronize(s));  // (`kern` is pageable and about to go out of scope)
    CU(ctx->ups_in.ensure((size_t)3 * f->xsize * f->ysize * 4));
    P.ups_kernel = (const float*)ctx->ups_kern.p;
  }
  ctx->sparse_used = 0;
  ctx->submitted.assign(ctx->num_groups, ctx->coeff_external ? 1 : 0);
  ctx->row_count.assign(P.yg, ctx->coeff_external ? P.xg : 0);
  ctx->row_bytes.assign(P.yg, 0);
  ctx->groups_in = 0;
  ctx->row_idct.assign(P.yg, 0);
  ctx->row_filtered.assign(P.yg, 0);
  if (P.yg > ctx->row_cap) {
    for (auto ev : ctx->row_events) cudaEventDestroy(ev);
    ctx->row_cap = P.yg;
    ctx->row_events.assign(ctx->row_cap, nullptr);
    for (auto& ev : ctx->row_events) CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  }
  ctx->row_event_used.assign(ctx->row_cap, 0);
  ctx->host_out = nullptr;
  ctx->host_out_stride = 0;
  ctx->stream_error = 0;
  ctx->in_frame = true;
  return JXLGPU_OK;
}

int jxlgpu_frame_set_output(jxlgpu_ctx* ctx, void* out, size_t out_stride_bytes) {
  if (!ctx) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (!ctx->in_frame) return JXLGPU_ERR_STATE;
  if (out && out_stride_bytes < ctx->out_row_bytes) return JXLGPU_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->host_out = out;
  ctx->host_out_stride = out_stride_bytes;
  return JXLGPU_OK;
}

// bookkeeping after the DMA(s) of group g were enqueued on the upload stream; ctx->mu is held
static int mark_submitted(jxlgpu_ctx* ctx, uint32_t g, size_t bytes) {
  const uint32_t row = g / ctx->P.xg;
  ctx->row_bytes[row] += bytes;
  cudaError_t e = cudaEventRecord(ctx->row_events[row], ctx->up_streams[0]);
  if (e != cudaSuccess) return fail_cuda(ctx, e, "cudaEventRecord(row)");
  ctx->row_event_used[row] = 1;
  if (ctx->submitted[g]) return JXLGPU_OK;  // a re-submission is not streamed again
  ctx->submitted[g] = 1;
  const bool needed = row >= ctx->need_row0 && row < ctx->need_row1;
  if (needed) ctx->groups_in++;
  if (++ctx->row_count[row] == ctx->P.xg && needed) {
    int rc = pump(ctx, false);
    if (rc) {
      ctx->stream_error = rc;
      return rc;
    }
  }
  return JXLGPU_OK;
}

static bool group_is_one_block(const void* const coeff[3], size_t es) {
  const uint8_t* c0 = (const uint8_t*)coeff[0];
  return (const uint8_t*)coeff[1] == c0 + 65536 * es && (const uint8_t*)coeff[2] == c0 + 2 * 65536 * es;
}

int jxlgpu_submit_groups(jxlgpu_ctx* ctx, size_t n, const uint32_t* group_idx, size_t thread_id,
                         const void* const* coeff, const size_t* ncoeff) {
  if (!ctx || !group_idx || !coeff || !ncoeff) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (!ctx->in_frame || ctx->coeff_external) return JXLGPU_ERR_STATE;
  if (thread_id >= ctx->num_threads) return JXLGPU_ERR_INVALID_ARGUMENT;
  for (size_t i = 0; i < n; i++) {
    if (group_idx[i] >= ctx->num_groups || ncoeff[i] > 65536) return JXLGPU_ERR_INVALID_ARGUMENT;
    for (int c = 0; c < 3; c++)
      if (!coeff[3 * i + c]) return JXLGPU_ERR_INVALID_ARGUMENT;
  }
  // NB: cudaSetDevice is per host thread
  cudaError_t e = cudaSetDevice(ctx->device);
  if (e != cudaSuccess) return JXLGPU_ERR_CUDA;
  // One FIFO upload stream for all host threads: DMAs complete in submission order, so the first
  // AC-group rows are on the device (and their kernels / D2H running) while later rows still
  // travel.  (Concurrent upload streams time-slice the copy engine and every row finishes late.)
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaStream_t s = ctx->up_streams[0];
  const size_t es = ctx->elem_size, gbytes = 3 * 65536 * es;
  size_t i = 0;
  while (i < n) {
    const uint32_t g = group_idx[i];
    uint8_t* dst = (uint8_t*)ctx->coeff.p + (size_t)g * gbytes;
    size_t j = i;
    if (group_is_one_block(coeff + 3 * i, es)) {
      // Extend over consecutive groups whose [3][65536] host blocks are adjacent: one DMA for the
      // whole run (a row of AC groups = tens of MB: full-duplex PCIe needs few, large copies).
      while (j + 1 < n && group_idx[j + 1] == group_idx[j] + 1 && group_is_one_block(coeff + 3 * (j + 1), es) &&
             (const uint8_t*)coeff[3 * (j + 1)] == (const uint8_t*)coeff[3 * j] + gbytes)
        j++;
      e = cudaMemcpyAsync(dst, coeff[3 * i], (j - i) * gbytes + (2 * 65536 + ncoeff[j]) * es,
                          cudaMemcpyHostToDevice, s);
      if (e != cudaSuccess) return fail_cuda(ctx, e, "cudaMemcpyAsync(coefficient groups)");
    } else {
      for (int c = 0; c < 3; c++) {
        e = cudaMemcpyAsync(dst + (size_t)c * 65536 * es, coeff[3 * i + c], ncoeff[i] * es, cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) return fail_cuda(ctx, e, "cudaMemcpyAsync(coefficients)");
      }
    }
    for (size_t k = i; k <= j; k++) {
      int rc = mark_submitted(ctx, group_idx[k], 3 * ncoeff[k] * es);
      if (rc) return rc;
    }
    i = j + 1;
  }
  return JXLGPU_OK;
}

int jxlgpu_submit_groups_sparse(jxlgpu_ctx* ctx, size_t n, const jxlgpu_sparse_group* groups, size_t thread_id) {
  if (!ctx || (n && !groups)) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (!ctx->in_frame || ctx->coeff_external) return JXLGPU_ERR_STATE;
  if (thread_id >= ctx->num_threads) return JXLGPU_ERR_INVALID_ARGUMENT;
  size_t words = 0;
  for (size_t i = 0; i < n; i++) {
    const jxlgpu_sparse_group& g = groups[i];
    if (g.group_idx >= ctx->num_groups) return JXLGPU_ERR_INVALID_ARGUMENT;
    for (int c = 0; c < 3; c++) {
      if (g.n16[c] > 65536 || g.n32[c] > 65536 || (g.n16[c] && !g.nz16[c]) || (g.n32[c] && !g.nz32[c]))
        return JXLGPU_ERR_INVALID_ARGUMENT;
      if (g.n32[c] && !ctx->P.ac_is32) return JXLGPU_ERR_INVALID_ARGUMENT;  // would not fit the int16 planes
      words += g.n16[c] + 2 * (size_t)g.n32[c] + 1;  // (+1: pair lists start on an 8-byte boundary)
    }
  }
  cudaError_t e = cudaSetDevice(ctx->device);
  if (e != cudaSuccess) return JXLGPU_ERR_CUDA;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaStream_t s = ctx->up_streams[0];  // the FIFO upload stream (see jxlgpu_submit_groups)
  const size_t es = ctx->elem_size, gelems = 3 * 65536, gbytes = gelems * es;
  // staging: worst case (every coefficient non-zero) is one word per coefficient + slack
  const size_t cap_words = (size_t)ctx->num_groups * (gelems + 8);
  // (DevBuf::ensure is a no-op when the capacity suffices; a context that decoded a small frame first
  // must grow the staging buffer for a larger one)
  e = ctx->sparse.ensure(cap_words * 4);
  if (e != cudaSuccess) return fail_cuda(ctx, e, "alloc(sparse staging)");
  if (ctx->sparse_used + words > cap_words) {
    ctx->last_error = "sparse lists larger than the dense planes: submit dense groups instead";
    return JXLGPU_ERR_INVALID_ARGUMENT;
  }
  // 1. zero-fill the dense planes of these groups (runs of consecutive groups in one memset).  Zero-fill
  //    and scatter run on the compute stream, so that the upload stream carries DMAs only and the
  //    next batch's lists travel while this one is expanded.
  cudaStream_t cs = ctx->stream;
  for (size_t i = 0; i < n;) {
    size_t j = i;
    while (j + 1 < n && groups[j + 1].group_idx == groups[j].group_idx + 1) j++;
    e = cudaMemsetAsync((uint8_t*)ctx->coeff.p + (size_t)groups[i].group_idx * gbytes, 0, (j - i + 1) * gbytes, cs);
    if (e != cudaSuccess) return fail_cuda(ctx, e, "cudaMemsetAsync(coefficient groups)");
    i = j + 1;
  }
  // 2. copy the lists; host arrays that follow each other in memory travel as one DMA
  std::vector<SparseSeg> segs;
  segs.reserve(6 * n);
  uint32_t* stage = (uint32_t*)ctx->sparse.p;
  const uint32_t* run_src = nullptr;
  size_t run_words = 0, run_dst = 0;
  auto flush = [&]() -> cudaError_t {
    if (!run_words) return cudaSuccess;
    cudaError_t r = cudaMemcpyAsync(stage + run_dst, run_src, run_words * 4, cudaMemcpyHostToDevice, s);
    run_words = 0;
    return r;
  };
  auto add = [&](const uint32_t* src, size_t nwords, uint32_t entries, uint32_t dst_off, uint32_t wide) -> cudaError_t {
    if (!entries) return cudaSuccess;
    const bool joins = run_words && src == run_src + run_words && (!wide || ((run_dst + run_words) % 2 == 0));
    if (!joins) {
      cudaError_t r = flush();
      if (r != cudaSuccess) return r;
      if (wide && ctx->sparse_used % 2) ctx->sparse_used++;
      run_src = src;
      run_dst = ctx->sparse_used;
    }
    segs.push_back(SparseSeg{(uint32_t)(run_dst + run_words), entries, dst_off, wide});
    run_words += nwords;
    ctx->sparse_used = run_dst + run_words;
    return cudaSuccess;
  };
  for (size_t i = 0; i < n; i++) {
    const jxlgpu_sparse_group& g = groups[i];
    for (int c = 0; c < 3; c++) {
      const uint32_t dst_off = (uint32_t)((size_t)g.group_idx * gelems + (size_t)c * 65536);
      if ((e = add(g.nz16[c], g.n16[c], g.n16[c], dst_off, 0)) != cudaSuccess) return fail_cuda(ctx, e, "cudaMemcpyAsync(sparse)");
      if ((e = add(g.nz32[c], 2 * (size_t)g.n32[c], g.n32[c], dst_off, 1)) != cudaSuccess) return fail_cuda(ctx, e, "cudaMemcpyAsync(sparse)");
    }
  }
  if ((e = flush()) != cudaSuccess) return fail_cuda(ctx, e, "cudaMemcpyAsync(sparse)");
  if (n) {
    cudaEvent_t ev = ctx->row_events[groups[0].group_idx / ctx->P.xg];
    if ((e = cudaEventRecord(ev, s)) != cudaSuccess || (e = cudaStreamWaitEvent(cs, ev, 0)) != cudaSuccess)
      return fail_cuda(ctx, e, "event(sparse lists)");
  }
  // 3. scatter into the dense planes
  for (size_t s0 = 0; s0 < segs.size(); s0 += kMaxSparseSegs) {
    SparseBatch B;
    const size_t cnt = std::min((size_t)kMaxSparseSegs, segs.size() - s0);
    uint32_t max_n = 1;
    for (size_t k = 0; k < cnt; k++) {
      B.seg[k] = segs[s0 + k];
      max_n = std::max(max_n, B.seg[k].n);
    }
    const dim3 grid(std::min<uint32_t>((max_n + 1023) / 1024, 16), (unsigned)cnt);
    if (ctx->P.ac_is32) sparse_expand_kernel<true><<<grid, 256, 0, cs>>>(B, stage, ctx->coeff.p);
    else sparse_expand_kernel<false><<<grid, 256, 0, cs>>>(B, stage, ctx->coeff.p);
    ctx->launches += 1;
  }
  if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(ctx, e, "sparse_expand_kernel");
  for (size_t i = 0; i < n; i++) {
    const jxlgpu_sparse_group& g = groups[i];
    size_t gw = 0;
    for (int c = 0; c < 3; c++) gw += g.n16[c] + 2 * (size_t)g.n32[c];
    int rc = mark_submitted(ctx, g.group_idx, gw * 4);
    if (rc) return rc;
  }
  return JXLGPU_OK;
}

int jxlgpu_submit_group(jxlgpu_ctx* ctx, uint32_t g, size_t thread_id, const void* const coeff[3], size_t ncoeff) {
  if (!coeff) return JXLGPU_ERR_INVALID_ARGUMENT;
  return jxlgpu_submit_groups(ctx, 1, &g, thread_id, coeff, &ncoeff);
}

int jxlgpu_set_device_coefficients(jxlgpu_ctx* ctx, const void* const dev_coeff[3]) {
  if (!ctx) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (!dev_coeff) {
    ctx->coeff_external = false;
    return JXLGPU_OK;
  }
  ctx->coeff_external = true;
  for (int c = 0; c < 3; c++) ctx->P.coeff[c] = dev_coeff[c];
  ctx->P.coeff_gstride = 65536;
  if (ctx->in_frame) {
    ctx->submitted.assign(ctx->num_groups, 1);
    ctx->row_count.assign(ctx->P.yg, ctx->P.xg);
  }
  return JXLGPU_OK;
}

static int render_device_on(jxlgpu_ctx* ctx, void* dev_out, size_t out_stride_bytes, cudaStream_t s);

int jxlgpu_render_device(jxlgpu_ctx* ctx, void* dev_out, size_t out_stride_bytes, void* cuda_stream) {
  if (!ctx) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (!ctx->in_frame) return JXLGPU_ERR_STATE;
  CU(cudaSetDevice(ctx->device));
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!coeff_planes_aligned(ctx)) return JXLGPU_ERR_INVALID_ARGUMENT;
  cudaStream_t s = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  if (cuda_stream) {  // side info was uploaded on the context stream
    CU(cudaEventRecord(ctx->ev_ext, ctx->stream));
    CU(cudaStreamWaitEvent(s, ctx->ev_ext, 0));
  }
  const int rc = render_device_on(ctx, dev_out, out_stride_bytes, s);
  if (cuda_stream && rc == JXLGPU_OK) {
    // the context's buffers (side information, work lists, XYB planes) are busy until this render has run:
    // the next frame_begin / render on another stream is ordered behind it
    CU(cudaEventRecord(ctx->ev_ext_done, s));
    ctx->ext_pending = true;
  }
  return rc;
}

static int render_device_on(jxlgpu_ctx* ctx, void* dev_out, size_t out_stride_bytes, cudaStream_t s) {
  const FrameDev& P = ctx->P;
  const uint32_t band_h = P.band_y1 - P.band_y0;
  char* o = (char*)dev_out;
  size_t stride = out_stride_bytes;
  if (!o) {
    int rc = ensure_out(ctx);
    if (rc) return rc;
    o = (char*)ctx->out.p;
    stride = ctx->out_row_bytes;
  } else if (stride % out_align(P.out_format) || (uintptr_t)o % out_align(P.out_format) ||
             stride < ctx->out_row_bytes) {
    return JXLGPU_ERR_INVALID_ARGUMENT;
  }
  if (P.nrep || P.mc) {
    // fused all-gather: the 8-byte vector stores to the replicas mirror the local byte offsets (all
    // bases 8-byte aligned), and the multicast mapping moves 4-byte granules (f32 layouts only)
    if ((uintptr_t)o % 8) return JXLGPU_ERR_INVALID_ARGUMENT;
    if (P.mc && P.out_format > JXLGPU_OUT_PLANAR_F32) return JXLGPU_ERR_UNSUPPORTED;
    // upsampled / noisy frames are finished by upsample_kernel, which writes the local buffer only
    if (P.ups || P.noise) return JXLGPU_ERR_UNSUPPORTED;
  }
  int rc = launch_idct(ctx, ctx->need_row0, ctx->need_row1, P.need_y0, P.need_y1, s);
  if (rc) return rc;
  if (P.ups || P.noise) {
    rc = launch_filter(ctx, P.band_y0, P.band_y1, P.band_y0, band_h, o, stride, s);
    return rc ? rc : launch_upsample(ctx, o, stride, s);
  }
  if (!P.nrep || P.mc || ctx->gather_in_kernel || use_fused(ctx))
    return launch_filter(ctx, P.band_y0, P.band_y1, P.band_y0, band_h, o, stride, s);
  // Gather through the copy engines: the band is filtered in row chunks; as soon as a chunk is finished its
  // rows travel to every peer's frame buffer (peer-mapped addresses, NVLink) on side streams while the SMs
  // filter the next chunk.  The kernels run without the replay instantiation.
  const uint32_t nrep = P.nrep;
  for (uint32_t q = 0; q < nrep; q++) {
    if (!ctx->rep_streams[q]) CU(cudaStreamCreateWithFlags(&ctx->rep_streams[q], cudaStreamNonBlocking));
    if (!ctx->ev_rep[q]) CU(cudaEventCreateWithFlags(&ctx->ev_rep[q], cudaEventDisableTiming));
  }
  for (int i = 0; i < 8; i++)
    if (!ctx->ev_chunk[i]) CU(cudaEventCreateWithFlags(&ctx->ev_chunk[i], cudaEventDisableTiming));
  uint32_t chunk_rows = (band_h / 4 + 7) & ~7u;
  if (chunk_rows < 256) chunk_rows = 256;
  char* rep[8];
  for (uint32_t q = 0; q < nrep; q++) rep[q] = P.rep[q];
  ctx->P.nrep = 0;  // (the kernels of this call do not replicate)
  const size_t planes = out_planes(P.out_format);
  int chunk = 0;
  for (uint32_t y0 = P.band_y0; y0 < P.band_y1 && !rc; y0 += chunk_rows, chunk++) {
    const uint32_t y1 = y0 + chunk_rows < P.band_y1 ? y0 + chunk_rows : P.band_y1;
    rc = launch_filter(ctx, y0, y1, P.band_y0, band_h, o, stride, s);
    if (rc) break;
    cudaEvent_t ev = ctx->ev_chunk[chunk & 7];
    CU(cudaEventRecord(ev, s));
    bool sm_ok = ctx->gather_sm && (uintptr_t)o % 16 == 0 && stride % 16 == 0;
    for (uint32_t q = 0; q < nrep; q++) sm_ok = sm_ok && (uintptr_t)rep[q] % 16 == 0;
    if (sm_ok) {  // one copy kernel per chunk and plane on a side stream: every peer at once, 16-byte stores
      cudaStream_t cs = ctx->rep_streams[0];
      CU(cudaStreamWaitEvent(cs, ev, 0));
      for (size_t pl = 0; pl < planes; pl++) {
        const size_t off = (pl * band_h + (y0 - P.band_y0)) * stride;
        PeerDst dst{};
        dst.n = nrep;
        for (uint32_t q = 0; q < nrep; q++) dst.p[q] = rep[q] + off;
        peer_copy_kernel<<<ctx->num_sms, 256, 0, cs>>>(o + off, dst, (size_t)(y1 - y0) * stride);
        ctx->launches += 1;
      }
      CU(cudaGetLastError());
      continue;
    }
    for (uint32_t q = 0; q < nrep; q++) {
      const uint32_t peer = (q + (uint32_t)chunk) % nrep;  // (start every chunk at a different peer)
      CU(cudaStreamWaitEvent(ctx->rep_streams[peer], ev, 0));
      for (size_t pl = 0; pl < planes; pl++) {
        const size_t off = (pl * band_h + (y0 - P.band_y0)) * stride;
        CU(cudaMemcpyAsync(rep[peer] + off, o + off, (size_t)(y1 - y0) * stride, cudaMemcpyDeviceToDevice,
                           ctx->rep_streams[peer]));
      }
    }
  }
  ctx->P.nrep = nrep;
  for (uint32_t q = 0; q < nrep && !rc; q++) {  // the caller's stream continues when every copy has landed
    CU(cudaEventRecord(ctx->ev_rep[q], ctx->rep_streams[q]));
    CU(cudaStreamWaitEvent(s, ctx->ev_rep[q], 0));
  }
  return rc;
}

int jxlgpu_frame_finish(jxlgpu_ctx* ctx, void* out, size_t out_stride_bytes) {
  if (!ctx) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (!ctx->in_frame) return JXLGPU_ERR_STATE;
  CU(cudaSetDevice(ctx->device));
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->stream_error) return ctx->stream_error;
    // every group of the band (+ halo rows) must have arrived
    for (uint32_t g = ctx->need_row0 * ctx->P.xg; g < ctx->need_row1 * ctx->P.xg; g++)
      if (!ctx->submitted[g]) {
        ctx->last_error = "missing group";
        return JXLGPU_ERR_STATE;
      }
    if (!coeff_planes_aligned(ctx)) return JXLGPU_ERR_INVALID_ARGUMENT;
    int rc = pump(ctx, true);  // whatever the scheduler still holds back, and device-resident coefficients
    if (rc) return rc;
    for (uint32_t g = ctx->band_row0; g < ctx->band_row1; g++)
      if (!ctx->row_filtered[g]) {
        ctx->last_error = "scheduler left a row unrendered";
        return JXLGPU_ERR_STATE;
      }
  }
  if (ctx->P.ups || ctx->P.noise) {  // every row is filtered: upsample / add noise, then the whole output travels
    int rc = launch_upsample(ctx, (char*)ctx->out.p, ctx->out_row_bytes, ctx->stream);
    if (rc) return rc;
    if (!out && ctx->host_out) {
      out = ctx->host_out;
      out_stride_bytes = ctx->host_out_stride;
    }
    ctx->host_out = nullptr;
  }
  if (out && out != ctx->host_out) {
    const uint32_t band_h = (ctx->P.ups || ctx->P.noise) ? ctx->P.out_hh : ctx->P.band_y1 - ctx->P.band_y0;
    const size_t row_bytes = ctx->out_row_bytes;
    if (out_stride_bytes < row_bytes) return JXLGPU_ERR_INVALID_ARGUMENT;
    const size_t planes = out_planes(ctx->P.out_format);
    CU(download_rows(out, out_stride_bytes, ctx->out.p, row_bytes, planes * band_h, ctx->stream));
  }
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaStreamSynchronize(ctx->s_down));
  ctx->in_frame = false;
  return JXLGPU_OK;
}

int jxlgpu_set_output_replicas(jxlgpu_ctx* ctx, uint32_t n, void* const* dev_ptrs, void* multicast_ptr) {
  if (!ctx || n > 8 || (n && !dev_ptrs)) return JXLGPU_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  for (uint32_t i = 0; i < n; i++)
    if ((uintptr_t)dev_ptrs[i] % 8) return JXLGPU_ERR_INVALID_ARGUMENT;
  if ((uintptr_t)multicast_ptr % 8) return JXLGPU_ERR_INVALID_ARGUMENT;
  ctx->P.nrep = multicast_ptr ? 0 : n;
  for (uint32_t i = 0; i < 8; i++) ctx->P.rep[i] = i < n ? (char*)dev_ptrs[i] : nullptr;
  ctx->P.mc = (char*)multicast_ptr;
  // the gather mechanism can be chosen per set of replicas (JXLGPU_GATHER: unset/ce = copy engines, sm =
  // peer_copy_kernel, kernel = replay inside the filter kernel); also read when the context is created
  if (n) {
    const char* ge = getenv("JXLGPU_GATHER");
    ctx->gather_in_kernel = ge && ge[0] == 'k';
    ctx->gather_sm = ge && ge[0] == 's';
  }
  return JXLGPU_OK;
}

int jxlgpu_device_output(jxlgpu_ctx* ctx, void** dev_ptr, size_t* stride_bytes) {
  if (!ctx || !dev_ptr || !stride_bytes) return JXLGPU_ERR_INVALID_ARGUMENT;
  *dev_ptr = ctx->out.p;
  *stride_bytes = ctx->out_row_bytes;
  return ctx->out.p ? JXLGPU_OK : JXLGPU_ERR_STATE;
}

int jxlgpu_device_xyb(jxlgpu_ctx* ctx, float** dev_ptr, size_t* plane_stride_floats, size_t* row_stride_floats) {
  if (!ctx || !dev_ptr) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (!ctx->xyb.p) return JXLGPU_ERR_STATE;
  CU(cudaSetDevice(ctx->device));
  std::lock_guard<std::mutex> lk(ctx->mu);
  // the renders keep the intermediate in 8x8 block tiles: hand out a row-major copy, made after the last
  // render (which may have run on the caller's stream) and complete on return
  const FrameDev& P = ctx->P;
  CU(ctx->xyb_rows.ensure(3 * P.plane_stride * sizeof(float)));
  if (ctx->ext_pending) CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_ext_done, 0));
  const size_t n4 = 3 * P.plane_stride / 4;
  const unsigned grid = (unsigned)std::min<size_t>((n4 + 255) / 256, (size_t)ctx->num_sms * 8);
  xyb_untile_kernel<<<grid, 256, 0, ctx->stream>>>(P, (float*)ctx->xyb_rows.p);
  CU(cudaGetLastError());
  ctx->launches += 1;
  CU(cudaStreamSynchronize(ctx->stream));
  *dev_ptr = (float*)ctx->xyb_rows.p;
  if (plane_stride_floats) *plane_stride_floats = P.plane_stride;
  if (row_stride_floats) *row_stride_floats = (size_t)P.xb * 8;
  return JXLGPU_OK;
}

int jxlgpu_synchronize(jxlgpu_ctx* ctx) {
  if (!ctx) return JXLGPU_ERR_INVALID_ARGUMENT;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaStreamSynchronize(ctx->s_down));
  return JXLGPU_OK;
}

uint64_t jxlgpu_launch_count(const jxlgpu_ctx* ctx) { return ctx ? ctx->launches.load() : 0; }

int jxlgpu_set_profiling(jxlgpu_ctx* ctx, int enable) {
  if (!ctx) return JXLGPU_ERR_INVALID_ARGUMENT;
  ctx->profile = enable != 0;
  return JXLGPU_OK;
}

int jxlgpu_kernel_times(jxlgpu_ctx* ctx, float ms[5]) {
  if (!ctx || !ms) return JXLGPU_ERR_INVALID_ARGUMENT;
  if (!ctx->profile) return JXLGPU_ERR_STATE;
  CU(cudaSetDevice(ctx->device));
  CU(cudaEventSynchronize(ctx->prof_ev[5]));
  for (int i = 0; i < 5; i++) CU(cudaEventElapsedTime(&ms[i], ctx->prof_ev[i], ctx->prof_ev[i + 1]));
  return JXLGPU_OK;
}

void* jxlgpu_alloc_pinned(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}

void jxlgpu_free_pinned(void* p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
