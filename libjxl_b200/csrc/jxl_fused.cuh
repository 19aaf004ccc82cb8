// jxl_fused.cuh -- the fused decode kernel of the VarDCT transform path for sm_90a:
//
//   coefficients (HBM) --TMA--> shared memory --dequant + IDCT--> pixel ring (shared memory)
//        --> Gaborish --> EPF0/1/2 --> XYB->RGB [--> sRGB] --> output rows (shared memory) --TMA--> HBM (+ peers)
//
// Nothing but the coefficients, the per-block side information and the finished pixels crosses HBM: the
// XYB intermediate of the two-kernel path (12 B/px written + 12 B/px read) stays on chip.
//
// Structure (one persistent CTA per SM, 16 warps):
//   * A CTA owns a vertical strip of 32 block columns (256 px: 30 output block columns + one halo block
//     column on each side, which it transforms redundantly instead of exchanging a rim through HBM) and
//     marches down the rows of a segment in STEPS of 4 rows.
//   * The stages form a software pipeline through rings of rows in shared memory.  In step k the IDCT
//     stage produces the 8x8-block row k/2 (even k), filter stage i works on the 4-row group k - 2(i+1):
//     every stage only reads rows that were finished in earlier steps, so one __syncthreads() per step
//     orders everything.
//   * Work inside a step is cut into warp items, handed out dynamically (one shared-memory atomic per
//     item): an IDCT item = four 8x8 blocks (8 lanes each, the arithmetic of idct8_kernel); a filter item =
//     one TILE of 8 columns x 4 rows (half an 8x8 block), lane = (column, row).  A tile never straddles an
//     8x8 block, so the EPF's per-block "sigma too small: skip" test (stage_epf.cc:121-128) is uniform
//     across the warp -- the row-streaming kernel (one warp = 32 columns = four blocks) executed the EPF
//     arithmetic with a third of its lanes masked off on real frames (ncu: 21 of 32 lanes active).
//   * Data movement uses the bulk-copy (TMA) unit: the coefficients of the next block row are fetched with
//     cp.async.bulk (global -> shared, mbarrier complete_tx) one step before they are needed, finished
//     output rows are written with cp.async.bulk (shared -> global) -- to this GPU's frame and, on a
//     multi-GPU run, to every peer's (the fused all-gather) -- so the SMs issue neither the loads nor the
//     stores of the bulk data.
//
// Varblocks larger than 8x8 are transformed by idct_mid_kernel / idct_large_kernel into the XYB planes
// first; the IDCT stage copies those pixels into the ring (kBmapCopy records of the plan kernel).
// Arithmetic (operation order, FMAs) is that of filter_strip_body / block8_item, i.e. the reference's.
#pragma once

namespace jxlb {

// (mbarrier + bulk-copy primitives: jxl_kernels.cuh)

// ---------------------------------------------------------------------------
// geometry
// ---------------------------------------------------------------------------
constexpr int kTBlocks = 32;              // block columns per strip (incl. one halo block column each side)
constexpr int kTOutBlocks = 30;
constexpr int kTOut = 8 * kTOutBlocks;    // output columns per strip
constexpr int kTLead = 8;                 // strip column of the first output column
constexpr int kTPitch = 264;              // floats per channel row; 3*264 = 24 (mod 32): the 4 rows of a tile hit disjoint banks
constexpr int kTRow = 3 * kTPitch;        // floats per ring row (X, Y, B)
constexpr int kTWarps = 16;
constexpr int kTThreads = 32 * kTWarps;
constexpr int kTPRows = 24;               // pixel ring: three block rows
constexpr int kTScratchWords = 200;       // per block: raw coefficients (3 x 64 int32 at most), then co/tmp of the transform
constexpr int kTStageRow = kTOut * 12;    // bytes of one staged output row (RGB f32 at most)
constexpr int kTPad = 8;                  // floats in front of the rings (tile 0 reads up to 3 columns to the left)

// filter stage kinds
enum : int { kStG = 1, kStE0 = 2, kStE1 = 3, kStE2 = 4, kStX = 5 };

template <uint32_t MASK>
struct TileCfg {
  static constexpr bool G = (MASK & 1) != 0, E0 = (MASK & 2) != 0, E1 = (MASK & 4) != 0, E2 = (MASK & 8) != 0;
  static constexpr bool XYB = (MASK & 16) != 0;
  static constexpr int nfilt = (G ? 1 : 0) + (E0 ? 1 : 0) + (E1 ? 1 : 0) + (E2 ? 1 : 0);
  static constexpr int nst = nfilt ? nfilt : 1;  // a pass-through stage emits when there is no filter
  static constexpr int H = (G ? 1 : 0) + (E0 ? 3 : 0) + (E1 ? 2 : 0) + (E2 ? 1 : 0);
  // stage i (pipeline order): kind, border
  __host__ __device__ static constexpr int kind(int i) {
    int n = 0;
    if (G) { if (n == i) return kStG; n++; }
    if (E0) { if (n == i) return kStE0; n++; }
    if (E1) { if (n == i) return kStE1; n++; }
    if (E2) { if (n == i) return kStE2; n++; }
    return kStX;
  }
  __host__ __device__ static constexpr int border_of(int k) { return k == kStG ? 1 : k == kStE0 ? 3 : k == kStE1 ? 2 : k == kStE2 ? 1 : 0; }
  __host__ __device__ static constexpr int border(int i) { return border_of(kind(i)); }
  // rows of stage i's INPUT ring: the pixel ring for stage 0, otherwise 12 + border (see the header)
  __host__ __device__ static constexpr int in_rows(int i) { return i == 0 ? kTPRows : 12 + border(i); }
  __host__ __device__ static constexpr int ring_off(int i) {  // in floats, from the start of the rings
    int o = 0;
    for (int j = 0; j < i; j++) o += in_rows(j) * kTRow;
    return o;
  }
  static constexpr int ring_floats = ring_off(nst);
  // halo still to be consumed after stage i
  __host__ __device__ static constexpr int rem(int i) {
    int r = 0;
    for (int j = i + 1; j < nst; j++) r += border(j);
    return r;
  }
  // shared memory layout (bytes)
  static constexpr size_t off_rings = 0;
  static constexpr size_t off_scratch = (size_t)(kTPad + ring_floats + kTPad) * 4;
  static constexpr size_t off_stage = off_scratch + (size_t)kTBlocks * kTScratchWords * 4;
  static constexpr size_t off_recs = off_stage + 2 * 4 * (size_t)kTStageRow;
  static constexpr size_t off_ctr = off_recs + kTBlocks * sizeof(uint4);
  static constexpr size_t off_bar = off_ctr + 16;
  static constexpr size_t kSmemBytes = off_bar + 16;
};

__device__ __forceinline__ int wrap_n(int s, int n) { return s >= n ? s - n : s; }
__device__ __forceinline__ int mod_n(int s, int n) { s %= n; return s < 0 ? s + n : s; }

// pixels of a block written straight into the pixel ring
struct Block8ToRing {
  static constexpr int kPitch = kTRow;
  static constexpr bool kGuardPx = true;
  static constexpr bool kDctRows = false;
  float* base;  // ring address of (row 0 of the block row, channel 0, first column of the block)
  __device__ __forceinline__ float* px(int c) const { return base + c * kTPitch; }
  __device__ __forceinline__ void dct_col(int c, int l, const float* u, bool active) const {
    if (active) {
      float* o = base + c * kTPitch + l;
#pragma unroll
      for (int y = 0; y < 8; y++) o[y * kTRow] = u[y];
    }
  }
  __device__ __forceinline__ void finish(int, int, bool) const { __syncwarp(); }
};

// XYB -> linear RGB (dec_xyb-inl.h:38-86)
__device__ __forceinline__ void xyb_to_rgb(const FrameDev& P, float& a, float& b, float& c3) {
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

// One pixel into a row segment whose pixel 0 sits at `row0` (shared-memory staging row, or the global row of
// the strip's first output column); `plane_bytes`: distance between the planes of the planar layout.
// (x, y): image coordinates (dither pattern).  The formats of store_px (stage_write.cc:455-640).
template <int OUTK>
__device__ __forceinline__ void store_px_at(const FrameDev& P, char* __restrict__ row0, size_t plane_bytes, int xi,
                                            int x, int y, float a, float b, float c3) {
  if constexpr (OUTK == 0) {
    float* o = reinterpret_cast<float*>(row0) + (size_t)xi * 3;
    o[0] = a; o[1] = b; o[2] = c3;
    return;
  }
  if (P.stage_mask & 32u) {
    a = srgb_from_linear(a);
    b = srgb_from_linear(b);
    c3 = srgb_from_linear(c3);
  }
  switch (P.out_format) {
    case 0: {
      float* o = reinterpret_cast<float*>(row0) + (size_t)xi * 3;
      o[0] = a; o[1] = b; o[2] = c3;
    } break;
    case 1: {
      reinterpret_cast<float*>(row0)[xi] = a;
      reinterpret_cast<float*>(row0 + plane_bytes)[xi] = b;
      reinterpret_cast<float*>(row0 + 2 * plane_bytes)[xi] = c3;
    } break;
    case 2: {
      uint8_t* o = reinterpret_cast<uint8_t*>(row0) + (size_t)xi * 3;
      o[0] = (uint8_t)make_unsigned<8>(a, x, y, 0);
      o[1] = (uint8_t)make_unsigned<8>(b, x, y, 1);
      o[2] = (uint8_t)make_unsigned<8>(c3, x, y, 2);
    } break;
    case 3: {
      const uint32_t w = make_unsigned<8>(a, x, y, 0) | (make_unsigned<8>(b, x, y, 1) << 8) |
                         (make_unsigned<8>(c3, x, y, 2) << 16) | 0xff000000u;
      reinterpret_cast<uint32_t*>(row0)[xi] = w;
    } break;
    case 4: {
      uint16_t* o = reinterpret_cast<uint16_t*>(row0) + (size_t)xi * 3;
      o[0] = (uint16_t)make_unsigned<16>(a, x, y, 0);
      o[1] = (uint16_t)make_unsigned<16>(b, x, y, 1);
      o[2] = (uint16_t)make_unsigned<16>(c3, x, y, 2);
    } break;
    default: {
      __half* o = reinterpret_cast<__half*>(row0) + (size_t)xi * 3;
      o[0] = __float2half_rn(a);
      o[1] = __float2half_rn(b);
      o[2] = __float2half_rn(c3);
    } break;
  }
}

// everything about one (strip, segment) work unit that the stage bodies need
struct TileUnit {
  int W, HI;            // image size
  int xs0;              // image column of strip column 0 (multiple of 8; -8 for the first strip)
  int x0;               // first output column
  int y_begin, y_end;   // output rows of the segment
  int ncols;            // output columns of the strip inside the image
  bool tma_out;         // finished rows leave through shared memory + cp.async.bulk (else: direct stores)
};

// ---------------------------------------------------------------------------
// filter stage bodies: one tile (8 columns x 4 rows), lane = (lx, ly).
//   in:  stage input ring (channel-0 plane of slot 0), `nin` rows; s0 = slot of row (4g - border)
//   EDGE: the tile needs mirroring / bounds checks (image border); otherwise no predicates at all.
// Each returns the filtered X, Y, B of the lane's pixel (row 4g + ly, strip column 8t + lx).
// ---------------------------------------------------------------------------
template <bool EDGE, int BORDER>
struct TileRows {
  // rowp[k]: pointer to (row 4g + ly - BORDER + k, channel 0, strip column of the lane) for k = 0 .. 2*BORDER
  const float* rowp[2 * BORDER + 1];
  int cn[2 * BORDER + 1];  // EDGE: column offsets of x - BORDER .. x + BORDER (mirrored), relative to the lane's column
  __device__ __forceinline__ float at(int k, int c, int d) const {  // row offset k - BORDER, channel c, column offset d - BORDER
    if constexpr (EDGE) return rowp[k][c * kTPitch + cn[d]];
    else return rowp[k][c * kTPitch + (d - BORDER)];
  }
};

// fast path: `off[k]` = float offset of (ring row of image row 4g + ly - BORDER + k, column lx), computed once per
// step; the tile only adds its first column
template <int BORDER>
__device__ __forceinline__ void tile_rows_fast(TileRows<false, BORDER>& R, const float* ring_col, const int* off) {
#pragma unroll
  for (int k = 0; k <= 2 * BORDER; k++) R.rowp[k] = ring_col + off[k];
}
// image border: rows and columns mirrored about the true image size (Mirror(), lib/jxl/image_ops.h:184-196)
template <int BORDER>
__device__ __forceinline__ void tile_rows_edge(TileRows<true, BORDER>& R, const TileUnit& U, const float* ring, int nin,
                                               int g, int col, int ly) {
  const int x = U.xs0 + col;
  const int r = 4 * g + ly;
#pragma unroll
  for (int k = 0; k <= 2 * BORDER; k++) R.rowp[k] = ring + mod_n(mirror_i(r - BORDER + k, U.HI), nin) * kTRow + col;
#pragma unroll
  for (int d = 0; d <= 2 * BORDER; d++) R.cn[d] = mirror_i(x - BORDER + d, U.W) - x;
}

// Gaborish (stage_gaborish.cc:56-100)
template <bool EDGE>
__device__ __forceinline__ void tile_gab(const FrameDev& P, const TileRows<EDGE, 1>& R, float* v) {
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float sum1 = (R.at(1, c, 0) + R.at(1, c, 2)) + (R.at(0, c, 1) + R.at(2, c, 1));
    const float sum2 = (R.at(0, c, 0) + R.at(0, c, 2)) + (R.at(2, c, 0) + R.at(2, c, 2));
    v[c] = fmaf(sum2, P.gab_w[3 * c + 2], fmaf(sum1, P.gab_w[3 * c + 1], R.at(1, c, 1) * P.gab_w[3 * c]));
  }
}

// EPF0 (stage_epf.cc:54-193): 12 neighbours, 5-pixel plus-window SADs
template <bool EDGE>
__device__ __forceinline__ void tile_epf0(const FrameDev& P, const TileRows<EDGE, 3>& R, float inv_sigma, float* v) {
  const int dy12[12] = {-2, -1, -1, -1, 0, 0, 0, 0, 1, 1, 1, 2};
  const int dx12[12] = {0, -1, 0, 1, -2, -1, 1, 2, -1, 0, 1, 0};
  const int py5[5] = {0, -1, 0, 1, 0};
  const int px5[5] = {0, 0, -1, 0, 1};
  float sads[12];
#pragma unroll
  for (int k = 0; k < 12; k++) sads[k] = 0.0f;
  float nbv[3][12];
  float ctr[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float w[7][7];  // the 25 pixels of the radius-3 diamond
#pragma unroll
    for (int a = 0; a < 7; a++)
#pragma unroll
      for (int b = 0; b < 7; b++)
        if ((a > 3 ? a - 3 : 3 - a) + (b > 3 ? b - 3 : 3 - b) <= 3) w[a][b] = R.at(a, c, b);
    ctr[c] = w[3][3];
    const float scale = P.epf_scale[c];
#pragma unroll
    for (int k = 0; k < 12; k++) {
      float sad = 0.0f;
#pragma unroll
      for (int o = 0; o < 5; o++) {
        // |a-b| == |b-a| exactly: subtract in (row, column) order so that equal pairs are shared
        const int a0 = 3 + py5[o], b0 = 3 + px5[o];
        const int a1 = a0 + dy12[k], b1 = b0 + dx12[k];
        const bool sw = (a1 < a0) || (a1 == a0 && b1 < b0);
        const float lhs = sw ? w[a1][b1] : w[a0][b0];
        const float rhs = sw ? w[a0][b0] : w[a1][b1];
        sad = sad + fabsf(lhs - rhs);
      }
      sads[k] = fmaf(sad, scale, sads[k]);
      nbv[c][k] = w[3 + dy12[k]][3 + dx12[k]];
    }
  }
  float wsum = 1.0f, X = ctr[0], Y = ctr[1], B = ctr[2];
#pragma unroll
  for (int k = 0; k < 12; k++) {
    const float wt = epf_weight(sads[k], inv_sigma);
    wsum = wsum + wt;
    X = fmaf(wt, nbv[0][k], X);
    Y = fmaf(wt, nbv[1][k], Y);
    B = fmaf(wt, nbv[2][k], B);
  }
  const float inv_w = 1.0f / wsum;
  v[0] = X * inv_w; v[1] = Y * inv_w; v[2] = B * inv_w;
}

// EPF1 (stage_epf.cc:197-379): 4 neighbours, plus-window SADs with the reference's accumulation order
template <bool EDGE>
__device__ __forceinline__ void tile_epf1(const FrameDev& P, const TileRows<EDGE, 2>& R, float inv_sigma, float* v) {
  float sad0 = 0.0f, sad1 = 0.0f, sad2 = 0.0f, sad3 = 0.0f;
  float nb[3][4], ctr[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float p20 = R.at(0, c, 2), p11 = R.at(1, c, 1), p21 = R.at(1, c, 2), p31 = R.at(1, c, 3);
    const float p02 = R.at(2, c, 0), p12 = R.at(2, c, 1), p22 = R.at(2, c, 2), p32 = R.at(2, c, 3), p42 = R.at(2, c, 4);
    const float p13 = R.at(3, c, 1), p23 = R.at(3, c, 2), p33 = R.at(3, c, 3), p24 = R.at(4, c, 2);
    nb[c][0] = p21; nb[c][1] = p12; nb[c][2] = p32; nb[c][3] = p23;
    ctr[c] = p22;
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
  float wsum = 1.0f, X = ctr[0], Y = ctr[1], B = ctr[2];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const float wt = epf_weight(sd[k], inv_sigma);
    wsum = wsum + wt;
    X = fmaf(wt, nb[0][k], X);
    Y = fmaf(wt, nb[1][k], Y);
    B = fmaf(wt, nb[2][k], B);
  }
  const float inv_w = 1.0f / wsum;
  v[0] = X * inv_w; v[1] = Y * inv_w; v[2] = B * inv_w;
}

// EPF2 (stage_epf.cc:383-506): 4 neighbours, single-pixel 3-channel SAD
template <bool EDGE>
__device__ __forceinline__ void tile_epf2(const FrameDev& P, const TileRows<EDGE, 1>& R, float inv_sigma, float* v) {
  const float rx = R.at(1, 0, 1), ry = R.at(1, 1, 1), rb = R.at(1, 2, 1);
  const int nk[4] = {0, 1, 1, 2};  // rows of N, W, E, S
  const int nd[4] = {1, 0, 2, 1};  // columns
  float wsum = 1.0f, X = rx, Y = ry, B = rb;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const float cx = R.at(nk[k], 0, nd[k]), cy = R.at(nk[k], 1, nd[k]), cb = R.at(nk[k], 2, nd[k]);
    float sad = fabsf(cx - rx) * P.epf_scale[0];
    sad = fmaf(fabsf(cy - ry), P.epf_scale[1], sad);
    sad = fmaf(fabsf(cb - rb), P.epf_scale[2], sad);
    const float wt = epf_weight(sad, inv_sigma);
    wsum = wsum + wt;
    X = fmaf(wt, cx, X);
    Y = fmaf(wt, cy, Y);
    B = fmaf(wt, cb, B);
  }
  const float inv_w = 1.0f / wsum;
  v[0] = X * inv_w; v[1] = Y * inv_w; v[2] = B * inv_w;
}

// ---------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------
// shared-space atomic (a generic-address atomicAdd costs ~40 instructions of address-space dispatch)
__device__ __forceinline__ int smem_fetch_add(int* p, int v) {
#if JXLB_PTX
  int old;
  asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(smem_addr(p)), "r"(v) : "memory");
  return old;
#else
  return atomicAdd(p, v);
#endif
}

constexpr int kTChunk = 2;                       // tiles per filter item
constexpr int kTChunks = kTBlocks / kTChunk;     // filter items per stage and step

template <uint32_t MASK, bool I32, int OUTK>
__global__ void __launch_bounds__(kTThreads, 1)
fused_tile_kernel(const __grid_constant__ FrameDev P, char* __restrict__ out, size_t out_row_stride, int seg_rows,
                  int strips, int units) {
  using C = TileCfg<MASK>;
  extern __shared__ __align__(16) float fsm[];
  char* smem = reinterpret_cast<char*>(fsm);
  float* rings = reinterpret_cast<float*>(smem + C::off_rings) + kTPad;
  uint32_t* scratch = reinterpret_cast<uint32_t*>(smem + C::off_scratch);
  char* stage = smem + C::off_stage;  // [2][4][kTStageRow]
  uint4* recs = reinterpret_cast<uint4*>(smem + C::off_recs);
  int* ctr = reinterpret_cast<int*>(smem + C::off_ctr);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + C::off_bar);

  const int tid = threadIdx.x, lane = tid & 31;
  const int lx = lane & 7, ly = lane >> 3;
  const float kMinSigma = -3.90524291751269967465540850526868f;
  const int pxb = out_pixel_bytes(P.out_format);
  const int band_h = (int)P.out_h;
  constexpr int H = C::H;
  constexpr int NST = C::nst;
  const bool lxborder = lx == 0 || lx == 7;

  if (tid == 0) {
    mbar_init(bar, 1);
    ctr[0] = ctr[1] = 0;
  }
  fence_async_smem();
  __syncthreads();
  uint32_t tma_phase = 0;  // parity of the coefficient barrier's next completion (uniform)

  // the rows a finished step left in the staging buffer `sb` (group g) leave through the TMA unit (thread 0)
  auto store_rows = [&](const TileUnit& U, int g, const char* sb) {
#pragma unroll 1
    for (int r = 0; r < 4; r++) {
      const int y = 4 * g + r;
      if (y < U.y_begin || y >= U.y_end) continue;
      const size_t yo = (size_t)(y - (int)P.out_y0);
      if (P.out_format == 1) {
#pragma unroll 1
        for (int c = 0; c < 3; c++) {
          const size_t off = ((size_t)c * band_h + yo) * out_row_stride + (size_t)U.x0 * 4;
          const char* src = sb + (size_t)r * kTStageRow + (size_t)c * kTOut * 4;
          bulk_s2g(out + off, src, (uint32_t)(U.ncols * 4));
#pragma unroll 1
          for (uint32_t q = 0; q < P.nrep; q++) bulk_s2g(P.rep[q] + off, src, (uint32_t)(U.ncols * 4));
        }
      } else {
        const size_t off = yo * out_row_stride + (size_t)U.x0 * pxb;
        const char* src = sb + (size_t)r * kTStageRow;
        bulk_s2g(out + off, src, (uint32_t)(U.ncols * pxb));
#pragma unroll 1
        for (uint32_t q = 0; q < P.nrep; q++) bulk_s2g(P.rep[q] + off, src, (uint32_t)(U.ncols * pxb));
      }
    }
    bulk_commit();
  };

#pragma unroll 1
  for (int unit = blockIdx.x; unit < units; unit += gridDim.x) {
    TileUnit U;
    U.W = (int)P.xsize;
    U.HI = (int)P.ysize;
    const int strip = unit % strips, seg = unit / strips;
    U.x0 = strip * kTOut;
    U.xs0 = U.x0 - kTLead;
    U.y_begin = (int)P.band_y0 + seg * seg_rows;
    U.y_end = min((int)P.band_y1, U.y_begin + seg_rows);
    U.ncols = min(kTOut, U.W - U.x0);
    // bulk stores need 16-byte aligned rows and sizes (the host checked base pointer and stride)
    U.tma_out = ((U.ncols * (P.out_format == 1 ? 4 : pxb)) & 15) == 0 && (P.fused & 2u);
    const int bx0 = U.xs0 >> 3;  // block column of strip column 0 (-1 for the first strip)

    // rows each stage must produce (stage i's output feeds rem(i) rows of halo) and the tiles of a stage that
    // need the slow path because of the left / right image border
    int lo[NST], hi[NST], t_lo[NST], t_hi[NST];
#pragma unroll
    for (int i = 0; i < NST; i++) {
      lo[i] = max(0, U.y_begin - C::rem(i));
      hi[i] = min(U.HI, U.y_end + C::rem(i));
      // fast iff xs0 + 8t - b >= 0 and xs0 + 8t + 7 + b < W
      t_lo[i] = U.xs0 < 0 ? 2 : 0;  // (xs0 = -8: tile 0 is outside, tile 1 touches column 0)
      t_hi[i] = (U.W - 8 - C::border(i) - U.xs0) >> 3;  // last fast tile (may be negative or >= kTBlocks)
      if (U.W - 8 - C::border(i) - U.xs0 < 0) t_hi[i] = -1;
    }
    const int lo_p = max(0, U.y_begin - H), hi_p = min(U.HI, U.y_end + H);
    const int B0 = lo_p >> 3, B1 = (hi_p - 1) >> 3;
    const int k_first = 2 * B0 - 1;
    const int k_last = ((hi[NST - 1] - 1) >> 2) + 2 * NST;
    int staged_k = -1000000;  // step whose output rows wait in the staging buffer (thread 0 bookkeeping)
    if (tid == 0) ctr[0] = ctr[1] = 0;
    __syncthreads();

#pragma unroll 1
    for (int k = k_first; k <= k_last; k++) {
      // ---- finished rows of the previous step leave through the TMA unit ----
      if (tid == 0 && U.tma_out && staged_k == k - 1) store_rows(U, (k - 1) - 2 * NST, stage + (size_t)((k - 1) & 1) * 4 * kTStageRow);

      // ---- per-step state, hoisted out of the items ----
      const bool prep_on = (k & 1) && ((k + 1) >> 1) >= B0 && ((k + 1) >> 1) <= B1;
      const bool idct_on = !(k & 1) && (k >> 1) >= B0 && (k >> 1) <= B1;
      const int base_filter = (idct_on ? kTBlocks / 4 : 0) + (prep_on ? 1 : 0);
      int n_items = base_filter;
      uint32_t amap = 0;                 // active filter stages, last first, 4 bits each
      bool edge_y[NST];
      int in_off[NST][7];                // per lane: ring offsets of the stage's input rows (fast path)
      int out_off[NST];                  // per lane: ring offset of the row the lane writes
      const float* sig_row[NST];
      float vsm[NST];
      {
        int slot = 0;
#pragma unroll
        for (int i = NST - 1; i >= 0; i--) {
          const int g = k - 2 * (i + 1);
          const bool on = g >= 0 && 4 * g + 3 >= lo[i] && 4 * g < hi[i];
          if (on) {
            amap |= (uint32_t)i << (4 * slot);
            slot++;
            n_items += kTChunks;
          }
          constexpr int b = 0;
          (void)b;
          const int B = C::border(i);
          const int NIN = C::in_rows(i);
          edge_y[i] = (4 * g - B < 0) || (4 * g + 3 + B >= U.HI);
          const int s0 = mod_n(4 * g - B, NIN) + ly;
#pragma unroll
          for (int q = 0; q < 7; q++)
            if (q <= 2 * B) in_off[i][q] = wrap_n(s0 + q, NIN) * kTRow + lx;
          if (i + 1 < NST) {
            const int NOUT = C::in_rows(i + 1 < NST ? i + 1 : i);
            out_off[i] = wrap_n(mod_n(4 * g, NOUT) + ly, NOUT) * kTRow + lx;
          } else {
            out_off[i] = 0;
          }
          const int KIND = C::kind(i);
          if (KIND == kStE0 || KIND == kStE1 || KIND == kStE2) {
            const int r = min(max(4 * g, 0), U.HI - 1);
            sig_row[i] = P.sigma + (size_t)(r >> 3) * P.xb + bx0;
            const int iy = (4 * g + ly) & 7;
            const float sm_ = P.epf_sm[KIND - kStE0];
            vsm[i] = (iy == 0 || iy == 7 || lxborder) ? sm_ * P.epf_border_mul : sm_;
          } else {
            sig_row[i] = nullptr;
            vsm[i] = 0.0f;
          }
        }
      }
      const bool emit_on = (amap & 15u) == (uint32_t)(NST - 1) && n_items > base_filter;
      if (emit_on && tid == 0) staged_k = k;
      char* stg_lane = stage + ((size_t)(k & 1) * 4 + ly) * kTStageRow;

      // ---- one filter tile ----
      auto tile = [&](auto itag, int t) {
        constexpr int I = decltype(itag)::value;
        constexpr int KIND = C::kind(I);
        constexpr int BORDER = C::border(I);
        constexpr int NIN = C::in_rows(I);
        constexpr bool LAST = I == NST - 1;
        const int g = k - 2 * (I + 1);
        const int r = 4 * g + ly;
        const int col = 8 * t + lx;
        const int x = U.xs0 + col;
        const float* in_ring = rings + C::ring_off(I);
        const bool edge = edge_y[I] || t < t_lo[I] || t > t_hi[I];
        float v[3];
        bool ok = true;  // the lane produces a pixel
        auto run = [&](auto edge_tag) {
          constexpr bool EDGE = decltype(edge_tag)::value;
          if constexpr (EDGE) ok = x >= 0 && x < U.W && r < U.HI;
          if (!ok) return;
          float s = 0.0f, inv_sigma = 0.0f;
          if constexpr (KIND == kStE0 || KIND == kStE1 || KIND == kStE2) {
            if constexpr (EDGE) {
              const int bxs = min(max(bx0 + t, 0), (int)P.xb - 1);
              s = __ldg(P.sigma + (size_t)(min(r, U.HI - 1) >> 3) * P.xb + bxs);
            } else {
              s = __ldg(sig_row[I] + t);
            }
            inv_sigma = s * vsm[I];
          }
          TileRows<EDGE, BORDER> R;
          if constexpr (KIND != kStX) {
            if constexpr (EDGE) tile_rows_edge(R, U, in_ring, NIN, g, col, ly);
            else tile_rows_fast(R, in_ring + 8 * t, in_off[I]);
          }
          if constexpr (KIND == kStG) {
            tile_gab(P, R, v);
          } else if constexpr (KIND == kStE0) {
            if (s < kMinSigma) { v[0] = R.at(3, 0, 3); v[1] = R.at(3, 1, 3); v[2] = R.at(3, 2, 3); }
            else tile_epf0(P, R, inv_sigma, v);
          } else if constexpr (KIND == kStE1) {
            if (s < kMinSigma) { v[0] = R.at(2, 0, 2); v[1] = R.at(2, 1, 2); v[2] = R.at(2, 2, 2); }
            else tile_epf1(P, R, inv_sigma, v);
          } else if constexpr (KIND == kStE2) {
            if (s < kMinSigma) { v[0] = R.at(1, 0, 1); v[1] = R.at(1, 1, 1); v[2] = R.at(1, 2, 1); }
            else tile_epf2(P, R, inv_sigma, v);
          } else {
            const float* p = in_ring + in_off[I][0] + 8 * t;
            v[0] = p[0]; v[1] = p[kTPitch]; v[2] = p[2 * kTPitch];
          }
        };
        if (edge) run(std::true_type());
        else run(std::false_type());
        if (!ok) return;
        if constexpr (!LAST) {
          float* o = rings + C::ring_off(I + 1) + out_off[I] + 8 * t;
          o[0] = v[0];
          o[kTPitch] = v[1];
          o[2 * kTPitch] = v[2];
        } else {
          if (r < U.y_begin || r >= U.y_end || x >= U.W) return;
          float a = v[0], b = v[1], c3 = v[2];
          if constexpr (C::XYB) xyb_to_rgb(P, a, b, c3);
          if (U.tma_out) {
            store_px_at<OUTK>(P, stg_lane, (size_t)kTOut * 4, col - kTLead, x, r, a, b, c3);
          } else {
            const size_t yo = (size_t)(r - (int)P.out_y0);
            if (P.out_format == 1)
              store_px_at<OUTK>(P, out + yo * out_row_stride + (size_t)U.x0 * 4, (size_t)band_h * out_row_stride,
                                col - kTLead, x, r, a, b, c3);
            else
              store_px_at<OUTK>(P, out + yo * out_row_stride + (size_t)U.x0 * pxb, 0, col - kTLead, x, r, a, b, c3);
          }
        }
      };
      auto chunk = [&](auto itag, int c) {
        constexpr int I = decltype(itag)::value;
        constexpr bool LAST = I == NST - 1;
#pragma unroll 1
        for (int q = 0; q < kTChunk; q++) {
          const int t = kTChunk * c + q;
          if (LAST && (t == 0 || t == kTBlocks - 1)) continue;  // halo block columns produce no output
          tile(itag, t);
        }
      };

#pragma unroll 1
      while (true) {
        int item = 0;
        if (lane == 0) item = smem_fetch_add(&ctr[k & 1], 1);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= n_items) break;
        if (item >= base_filter) {
          const int fi = item - base_filter;
          const int si = (int)((amap >> (4 * (fi / kTChunks))) & 15u);
          const int c = fi % kTChunks;
          if (si == 0) chunk(IC<0>(), c);
          if constexpr (NST > 1) { if (si == 1) chunk(IC<1>(), c); }
          if constexpr (NST > 2) { if (si == 2) chunk(IC<2>(), c); }
          if constexpr (NST > 3) { if (si == 3) chunk(IC<3>(), c); }
          continue;
        }
        if (idct_on) {
          // =================== IDCT item: ranks 4*item .. 4*item+3 of block row B ===================
          const int B = k >> 1;
          const int slot = lane >> 3, l = lane & 7;
          const int rank = 4 * item + slot;
          mbar_wait(bar, tma_phase);
          const uint4 rec = recs[rank];
          const int kind = (int)(rec.x & 0xffu), bxl = (int)((rec.x >> 8) & 0xffu);
          uint32_t* stg = scratch + rank * kTScratchWords;
          float* scr = reinterpret_cast<float*>(stg);
          Block8ToRing ro;
          ro.base = rings + (size_t)((B % 3) * 8) * kTRow + bxl * 8;
          float val[3][8];
          const bool inl = kind < (int)kBmapSkip;
          if (inl) {
            VarblockCtx vb;
            vb.abx = (uint32_t)(bx0 + bxl);
            vb.aby = (uint32_t)B;
            vb.cbase = 0;
            const float s = P.inv_global_scale / (float)(int)rec.z;
            vb.sx = s * P.x_dm;
            vb.sy = s;
            vb.sb = s * P.b_dm;
            vb.x_cc = P.cfl_base_x + (float)(int)(int8_t)(rec.w & 0xffu) * P.cfl_scale;
            vb.b_cc = P.cfl_base_b + (float)(int)(int8_t)((rec.w >> 8) & 0xffu) * P.cfl_scale;
            constexpr int kChWords = I32 ? 64 : 32;
            const bool col = kind == 0;  // (per slot: the slots of an item may hold different kinds)
            block8_dequant(P, kind, vb, l, col,
                           [&](int c, int* q) { load_lane8_smem<I32>(stg + c * kChWords, l, col, q); }, val);
          } else {
#pragma unroll
            for (int c = 0; c < 3; c++)
#pragma unroll
              for (int e = 0; e < 8; e++) val[c][e] = 0.0f;
          }
          __syncwarp();  // every lane holds its row: the staging words become the transform's scratch
          // the (at most four) distinct kinds of the warp's slots, one after the other
          uint32_t done = 0;
#pragma unroll 1
          for (int sidx = 0; sidx < 4; sidx++) {
            if ((done >> sidx) & 1u) continue;
            const int kc = __shfl_sync(0xffffffffu, kind, 8 * sidx);
            const bool act = kind == kc;
            const uint32_t m = __ballot_sync(0xffffffffu, act);
            done |= (m & 1u) | ((m >> 7) & 2u) | ((m >> 14) & 4u) | ((m >> 21) & 8u);
            if (kc == (int)kBmapSkip) continue;
            if (kc == (int)kBmapCopy) {
              if (act) {  // lane l copies pixel row l of the block from the XYB planes
                const float* src = P.xyb_block(0, B, bx0 + bxl) + l * 8;
#pragma unroll
                for (int c = 0; c < 3; c++) {
                  const float4 a = __ldg(reinterpret_cast<const float4*>(src + (size_t)c * P.plane_stride));
                  const float4 b = __ldg(reinterpret_cast<const float4*>(src + (size_t)c * P.plane_stride) + 1);
                  float* d = ro.base + (size_t)l * kTRow + c * kTPitch;
                  *reinterpret_cast<float4*>(d) = a;
                  *reinterpret_cast<float4*>(d + 4) = b;
                }
              }
              continue;
            }
            block8_transform(kc, act, val, l, scr, ro);
          }
          fence_async_smem();  // the scratch is the TMA destination of the next block row
        } else {
          // =================== PREP item: block row B's records, sorted by kind; its coefficients ===================
          const int B = (k + 1) >> 1;
          const int abx = bx0 + lane;
          uint4 rec = make_uint4(kBmapSkip, 0u, 1u, 0u);
          if (abx >= 0 && abx < (int)P.xb && B < (int)P.yb) rec = __ldg(P.bmap + (size_t)B * P.xb + abx);
          const int kind = (int)(rec.x & 0xffu);
          // sort key: the kinds in the order of idct8_kernel's lists, then copies, then nothing
          const int cls = kind == 0 ? 0 : kind == 2 ? 1 : kind == 12 ? 2 : kind == 13 ? 3 : kind == 1 ? 4 : kind == 3 ? 5
                        : (kind >= 14 && kind <= 17) ? kind - 8 : kind == (int)kBmapCopy ? 10 : 11;
          int below = 0, within = 0;
#pragma unroll
          for (int q = 0; q < 12; q++) {
            const uint32_t m = __ballot_sync(0xffffffffu, cls == q);
            if (q < cls) below += __popc(m);
            if (q == cls) within = __popc(m & ((1u << lane) - 1u));
          }
          const int rank = below + within;
          rec.x = (uint32_t)kind | ((uint32_t)lane << 8);
          recs[rank] = rec;
          const bool inl = kind < (int)kBmapSkip;
          const uint32_t ninl = __popc(__ballot_sync(0xffffffffu, inl));
          constexpr uint32_t kChBytes = I32 ? 256 : 128;
          if (lane == 0) mbar_arrive_expect_tx(bar, ninl * 3 * kChBytes);
          __syncwarp();
          if (inl) {
            char* dst = reinterpret_cast<char*>(scratch + rank * kTScratchWords);
            const size_t e0 = (size_t)rec.y * 64u * (I32 ? 4 : 2);
#pragma unroll
            for (int c = 0; c < 3; c++)
              bulk_g2s(dst + c * kChBytes, reinterpret_cast<const char*>(P.coeff[c]) + e0, kChBytes, bar);
          }
        }
      }
      // ---- end of step ----
      if (emit_on && U.tma_out) fence_async_smem();  // staged rows -> visible to the TMA unit
      if (tid == 0) {
        ctr[(k + 1) & 1] = 0;
        bulk_wait_read_all();  // the rows staged two steps ago have left: their buffer is written next step
      }
      if (idct_on) tma_phase ^= 1u;
      __syncthreads();
    }
    // the last step's rows
    if (tid == 0 && U.tma_out && staged_k == k_last) {
      store_rows(U, k_last - 2 * NST, stage + (size_t)(k_last & 1) * 4 * kTStageRow);
      bulk_wait_read_all();
    }
    __syncthreads();
  }
  if (tid == 0) bulk_wait_all();
}

}  // namespace jxlb
