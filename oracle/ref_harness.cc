// TEST INFRASTRUCTURE ONLY -- never linked into, loaded by, or called from the
// product library (libjxl_b200/csrc).  See oracle/README.md.
//
// A thin C ABI over the UNMODIFIED reference (libjxl 0.13.0 compiled by
// oracle/build_ref.py from /root/reference) so that tests and bench.py can
//   (1) manufacture VarDCT bitstreams (public JxlEncoder API),
//   (2) run the reference decoder end to end (public JxlDecoder API) -> linear
//       sRGB float pixels: the image-level oracle and the "full decode" CPU
//       baseline,
//   (3) open a frame with the reference's own FrameDecoder and keep the
//       entropy-decoded quantized coefficients + every side-info plane the hot
//       path consumes: exactly the hand-off SURVEY.md §8(b) describes,
//   (4) re-run ONLY the hot path (DecodeGroupForRoundtrip + the reference
//       render-pipeline stages) from those coefficients: stage-by-stage golden
//       images for the C restatement, and the transform-only CPU baseline,
//   (5) call the function-level facade the reference's own ac_strategy_test
//       uses (TransformToPixels / LowestFrequenciesFromDC).
//
// This file is OUR code; it only #includes reference headers.
// Flow of (3) mirrors jxl::DecodeFrame (lib/jxl/dec_frame.cc:82-133) with the
// sections fed in two ProcessSections calls so that accumulate-mode coefficient
// storage (lib/jxl/dec_group.cc:219,335-338) can be switched on in between.

#include <jxl/decode.h>
#include <jxl/encode.h>
#include <jxl/thread_parallel_runner.h>

#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <memory>
#include <vector>

#include "hwy/detect_targets.h"
#include "hwy/targets.h"
#include "lib/jxl/ac_strategy.h"
#include "lib/jxl/base/data_parallel.h"
#include "lib/jxl/base/span.h"
#include "lib/jxl/chroma_from_luma.h"
#include "../integration/gpu_frame_binding.h"
#include "../integration/pinned_ac_image.h"
#include "lib/jxl/color_encoding_internal.h"
#include "lib/jxl/compressed_dc.h"
#include "lib/jxl/modular/modular_image.h"
#include "lib/jxl/dct_util.h"
#include "lib/jxl/dec_bit_reader.h"
#include "lib/jxl/dec_cache.h"
#include "lib/jxl/dec_frame.h"
#include "lib/jxl/dec_group.h"
#include "lib/jxl/dec_transforms_testonly.h"
#include "lib/jxl/enc_aux_out.h"
#include "lib/jxl/enc_bit_writer.h"
#include "lib/jxl/enc_transforms.h"
#include "lib/jxl/epf.h"
#include "lib/jxl/fields.h"
#include "lib/jxl/frame_header.h"
#include "lib/jxl/headers.h"
#include "lib/jxl/image.h"
#include "lib/jxl/image_bundle.h"
#include "lib/jxl/image_metadata.h"
#include "lib/jxl/loop_filter.h"
#include "lib/jxl/memory_manager_internal.h"
#include "lib/jxl/passes_state.h"
#include "lib/jxl/quant_weights.h"
#include "lib/jxl/quantizer.h"
#include "lib/jxl/render_pipeline/render_pipeline.h"
#include "lib/jxl/render_pipeline/stage_epf.h"
#include "lib/jxl/render_pipeline/stage_from_linear.h"
#include "lib/jxl/dec_noise.h"
#include "lib/jxl/render_pipeline/stage_gaborish.h"
#include "lib/jxl/render_pipeline/stage_noise.h"
#include "lib/jxl/render_pipeline/stage_upsampling.h"
#include "lib/jxl/render_pipeline/stage_write.h"
#include "lib/jxl/render_pipeline/stage_xyb.h"
#include "lib/jxl/render_pipeline/stage_ycbcr.h"

#define REF_API extern "C" __attribute__((visibility("default")))

namespace {

double NowSec() {
  using namespace std::chrono;
  return duration<double>(steady_clock::now().time_since_epoch()).count();
}

struct Runner {
  explicit Runner(int threads) {
    opaque = JxlThreadParallelRunnerCreate(nullptr, threads < 1 ? 1 : threads);
  }
  ~Runner() { JxlThreadParallelRunnerDestroy(opaque); }
  void* opaque;
};

}  // namespace

// ---------------------------------------------------------------------------
// (1) encoder
// ---------------------------------------------------------------------------
REF_API void ref_free(void* p) { free(p); }

// gaborish / epf: -1 keeps the encoder default for the distance
// (lib/jxl/enc_frame.cc:316-341).  Output: bare codestream, malloc'd.
REF_API int ref_encode_rgb8_ex(const uint8_t* rgb, int w, int h, float distance, int effort, int gaborish, int epf,
                               int resampling, int threads, uint8_t** out, size_t* out_size);
REF_API int ref_encode_rgb8(const uint8_t* rgb, int w, int h, float distance,
                            int effort, int gaborish, int epf, int threads,
                            uint8_t** out, size_t* out_size) {
  return ref_encode_rgb8_ex(rgb, w, h, distance, effort, gaborish, epf, -1, threads, out, out_size);
}
// resampling: -1 = encoder default, 1/2/4/8 = JXL_ENC_FRAME_SETTING_RESAMPLING (frame_header.upsampling);
// + 256: JXL_ENC_FRAME_SETTING_PROGRESSIVE_AC (multi-pass frame); + (iso / 100) << 16: JXL_ENC_FRAME_SETTING_PHOTON_NOISE
REF_API int ref_encode_rgb8_ex(const uint8_t* rgb, int w, int h, float distance, int effort, int gaborish, int epf,
                               int resampling, int threads, uint8_t** out, size_t* out_size) {
  Runner runner(threads);
  JxlEncoder* enc = JxlEncoderCreate(nullptr);
  if (!enc) return 1;
  int rc = 0;
  std::vector<uint8_t> buf(1 << 20);
  do {
    if (JxlEncoderSetParallelRunner(enc, JxlThreadParallelRunner,
                                    runner.opaque) != JXL_ENC_SUCCESS) { rc = 2; break; }
    JxlEncoderUseContainer(enc, JXL_FALSE);
    JxlBasicInfo info;
    JxlEncoderInitBasicInfo(&info);
    info.xsize = w;
    info.ysize = h;
    info.bits_per_sample = 8;
    info.exponent_bits_per_sample = 0;
    info.num_color_channels = 3;
    info.num_extra_channels = 0;
    info.alpha_bits = 0;
    info.uses_original_profile = JXL_FALSE;
    if (JxlEncoderSetBasicInfo(enc, &info) != JXL_ENC_SUCCESS) { rc = 3; break; }
    JxlColorEncoding ce;
    JxlColorEncodingSetToSRGB(&ce, JXL_FALSE);
    if (JxlEncoderSetColorEncoding(enc, &ce) != JXL_ENC_SUCCESS) { rc = 4; break; }
    JxlEncoderFrameSettings* fs = JxlEncoderFrameSettingsCreate(enc, nullptr);
    JxlEncoderSetFrameDistance(fs, distance);
    JxlEncoderFrameSettingsSetOption(fs, JXL_ENC_FRAME_SETTING_EFFORT, effort);
    if (gaborish >= 0)
      JxlEncoderFrameSettingsSetOption(fs, JXL_ENC_FRAME_SETTING_GABORISH, gaborish);
    if (epf >= 0)
      JxlEncoderFrameSettingsSetOption(fs, JXL_ENC_FRAME_SETTING_EPF, epf);
    if (resampling > 0)
      JxlEncoderFrameSettingsSetOption(fs, JXL_ENC_FRAME_SETTING_RESAMPLING, resampling & 15);
    if (resampling > 0 && (resampling & 256))  // bit 8: progressive AC (several passes per group)
      JxlEncoderFrameSettingsSetOption(fs, JXL_ENC_FRAME_SETTING_PROGRESSIVE_AC, 1);
    if (resampling > 0 && (resampling >> 16))  // bits 16..: photon noise ISO / 100 (frame flag kNoise)
      JxlEncoderFrameSettingsSetFloatOption(fs, JXL_ENC_FRAME_SETTING_PHOTON_NOISE, 100.0f * (resampling >> 16));
    JxlPixelFormat pf = {3, JXL_TYPE_UINT8, JXL_NATIVE_ENDIAN, 0};
    if (JxlEncoderAddImageFrame(fs, &pf, rgb, static_cast<size_t>(w) * h * 3) !=
        JXL_ENC_SUCCESS) { rc = 5; break; }
    JxlEncoderCloseInput(enc);
    size_t pos = 0;
    for (;;) {
      uint8_t* next = buf.data() + pos;
      size_t avail = buf.size() - pos;
      JxlEncoderStatus st = JxlEncoderProcessOutput(enc, &next, &avail);
      pos = next - buf.data();
      if (st == JXL_ENC_NEED_MORE_OUTPUT) { buf.resize(buf.size() * 2); continue; }
      if (st != JXL_ENC_SUCCESS) rc = 6;
      break;
    }
    if (rc) break;
    *out = static_cast<uint8_t*>(malloc(pos));
    memcpy(*out, buf.data(), pos);
    *out_size = pos;
  } while (false);
  JxlEncoderDestroy(enc);
  return rc;
}

// (1b) lossless JPEG recompression (JxlEncoderAddJPEGFrame): a VarDCT frame with the YCbCr colour transform whose
// coefficients are the JPEG's own.  No reconstruction metadata is stored (pixels only).
REF_API int ref_encode_jpeg(const uint8_t* jpeg, size_t n, int threads, uint8_t** out, size_t* out_size) {
  Runner runner(threads);
  JxlEncoder* enc = JxlEncoderCreate(nullptr);
  if (!enc) return 1;
  int rc = 0;
  std::vector<uint8_t> buf(1 << 20);
  do {
    if (JxlEncoderSetParallelRunner(enc, JxlThreadParallelRunner, runner.opaque) != JXL_ENC_SUCCESS) { rc = 2; break; }
    JxlEncoderUseContainer(enc, JXL_FALSE);
    JxlEncoderStoreJPEGMetadata(enc, JXL_FALSE);
    JxlEncoderFrameSettings* fs = JxlEncoderFrameSettingsCreate(enc, nullptr);
    if (JxlEncoderAddJPEGFrame(fs, jpeg, n) != JXL_ENC_SUCCESS) { rc = 5; break; }
    JxlEncoderCloseInput(enc);
    size_t pos = 0;
    for (;;) {
      uint8_t* next = buf.data() + pos;
      size_t avail = buf.size() - pos;
      JxlEncoderStatus st = JxlEncoderProcessOutput(enc, &next, &avail);
      pos = next - buf.data();
      if (st == JXL_ENC_NEED_MORE_OUTPUT) { buf.resize(buf.size() * 2); continue; }
      if (st != JXL_ENC_SUCCESS) rc = 6;
      break;
    }
    if (rc) break;
    *out = static_cast<uint8_t*>(malloc(pos));
    memcpy(*out, buf.data(), pos);
    *out_size = pos;
  } while (false);
  JxlEncoderDestroy(enc);
  return rc;
}

// ---------------------------------------------------------------------------
// (2) full reference decode through the public API -> interleaved linear sRGB f32
// (same output djxl --color_space=RGB_D65_SRG_Rel_Lin produces; SURVEY §8c)
// `runner_opaque` may be NULL (a runner with `threads` workers is made).
// ---------------------------------------------------------------------------
REF_API void* ref_runner_create(int threads) {
  return JxlThreadParallelRunnerCreate(nullptr, threads < 1 ? 1 : threads);
}
REF_API void ref_runner_destroy(void* r) { JxlThreadParallelRunnerDestroy(r); }

REF_API int ref_decode_linear_f32(const uint8_t* jxl, size_t n, void* runner_opaque,
                                  int threads, float* out, size_t out_floats,
                                  int* w, int* h) {
  std::unique_ptr<Runner> own;
  if (!runner_opaque) { own.reset(new Runner(threads)); runner_opaque = own->opaque; }
  JxlDecoder* dec = JxlDecoderCreate(nullptr);
  if (!dec) return 1;
  int rc = 0;
  JxlPixelFormat pf = {3, JXL_TYPE_FLOAT, JXL_NATIVE_ENDIAN, 0};
  do {
    if (JxlDecoderSetParallelRunner(dec, JxlThreadParallelRunner, runner_opaque) !=
        JXL_DEC_SUCCESS) { rc = 2; break; }
    JxlDecoderSubscribeEvents(dec, JXL_DEC_BASIC_INFO | JXL_DEC_COLOR_ENCODING |
                                       JXL_DEC_FULL_IMAGE);
    JxlDecoderSetInput(dec, jxl, n);
    JxlDecoderCloseInput(dec);
    for (;;) {
      JxlDecoderStatus st = JxlDecoderProcessInput(dec);
      if (st == JXL_DEC_BASIC_INFO) {
        JxlBasicInfo info;
        JxlDecoderGetBasicInfo(dec, &info);
        *w = info.xsize;
        *h = info.ysize;
      } else if (st == JXL_DEC_COLOR_ENCODING) {
        JxlColorEncoding ce;
        JxlColorEncodingSetToLinearSRGB(&ce, JXL_FALSE);
        if (JxlDecoderSetOutputColorProfile(dec, &ce, nullptr, 0) != JXL_DEC_SUCCESS) {
          rc = 3; break;
        }
      } else if (st == JXL_DEC_NEED_IMAGE_OUT_BUFFER) {
        size_t need = 0;
        JxlDecoderImageOutBufferSize(dec, &pf, &need);
        if (!out) { rc = -1; break; }  // size query only
        if (need > out_floats * sizeof(float)) { rc = 4; break; }
        JxlDecoderSetImageOutBuffer(dec, &pf, out, need);
      } else if (st == JXL_DEC_FULL_IMAGE) {
        continue;
      } else if (st == JXL_DEC_SUCCESS) {
        break;
      } else { rc = 10 + static_cast<int>(st); break; }
    }
  } while (false);
  JxlDecoderDestroy(dec);
  return rc == -1 ? 0 : rc;
}

// (2b) public API, the way djxl decodes by default: no output colour profile override (an sRGB image
// comes out sRGB-encoded), caller-chosen JxlPixelFormat: data_type 0 = FLOAT, 2 = UINT8, 3 = UINT16,
// 5 = FLOAT16 (jxl/types.h:35-60), num_channels 3 or 4.  out_bytes = capacity of out.
REF_API int ref_decode_native(const uint8_t* jxl, size_t n, int threads, int data_type, int num_channels,
                              void* out, size_t out_bytes, int* w, int* h) {
  Runner runner(threads);
  JxlDecoder* dec = JxlDecoderCreate(nullptr);
  if (!dec) return 1;
  int rc = 0;
  JxlPixelFormat pf = {static_cast<uint32_t>(num_channels), static_cast<JxlDataType>(data_type), JXL_NATIVE_ENDIAN, 0};
  do {
    if (JxlDecoderSetParallelRunner(dec, JxlThreadParallelRunner, runner.opaque) != JXL_DEC_SUCCESS) { rc = 2; break; }
    JxlDecoderSubscribeEvents(dec, JXL_DEC_BASIC_INFO | JXL_DEC_FULL_IMAGE);
    JxlDecoderSetInput(dec, jxl, n);
    JxlDecoderCloseInput(dec);
    for (;;) {
      JxlDecoderStatus st = JxlDecoderProcessInput(dec);
      if (st == JXL_DEC_BASIC_INFO) {
        JxlBasicInfo info;
        JxlDecoderGetBasicInfo(dec, &info);
        *w = info.xsize;
        *h = info.ysize;
      } else if (st == JXL_DEC_NEED_IMAGE_OUT_BUFFER) {
        size_t need = 0;
        JxlDecoderImageOutBufferSize(dec, &pf, &need);
        if (need > out_bytes) { rc = 4; break; }
        JxlDecoderSetImageOutBuffer(dec, &pf, out, need);
      } else if (st == JXL_DEC_FULL_IMAGE) {
        continue;
      } else if (st == JXL_DEC_SUCCESS) {
        break;
      } else { rc = 10 + static_cast<int>(st); break; }
    }
  } while (false);
  JxlDecoderDestroy(dec);
  return rc;
}

// ---------------------------------------------------------------------------
// (3) frame opened with reference internals, coefficients retained
// ---------------------------------------------------------------------------
namespace {
using namespace jxl;

struct RefFrame {
  JxlMemoryManager mm;
  CodecMetadata metadata;
  std::unique_ptr<PassesDecoderState> dec_state;
  std::unique_ptr<ImageBundle> decoded;
  std::unique_ptr<FrameHeader> frame_header;
  void* runner = nullptr;
  std::unique_ptr<ThreadPool> pool;
  jxlb_integration::GpuFrameBinding binding;  // integration/gpu_frame_binding.h, see ref_frame_bind_gpu_frame
  int storage = 0;            // 0: ACImageT (reference), 1: integration/pinned_ac_image.h
  void* raw_base = nullptr;   // storage 1: the group-major allocation
  size_t raw_bytes = 0;
  // int32 copy of the coefficients for DecodeGroupForRoundtrip
  // (GetBlockFromEncoder requires k32: lib/jxl/dec_group.cc:668).
  std::vector<std::unique_ptr<ACImage>> ac32;
  // what the entropy decoder produced (int16 or int32, per dec_frame.cc:417-431)
  std::unique_ptr<ACImage> stored;
  bool is16 = false;
  uint32_t passes_shift_backup[kMaxNumPasses];
  ~RefFrame() {
    pool.reset();
    if (runner) JxlThreadParallelRunnerDestroy(runner);
  }
};

Status OpenImpl(RefFrame* f, const uint8_t* data, size_t n) {
  JXL_RETURN_IF_ERROR(MemoryManagerInit(&f->mm, nullptr));
  if (n < 2 || data[0] != 0xff || data[1] != kCodestreamMarker)
    return JXL_FAILURE("not a bare codestream");
  BitReader br(Bytes(data + 2, n - 2));
  Status ok = [&]() -> Status {
    JXL_RETURN_IF_ERROR(Bundle::Read(&br, &f->metadata.size));
    JXL_RETURN_IF_ERROR(Bundle::Read(&br, &f->metadata.m));
    f->metadata.transform_data.nonserialized_xyb_encoded = f->metadata.m.xyb_encoded;
    JXL_RETURN_IF_ERROR(Bundle::Read(&br, &f->metadata.transform_data));
    if (f->metadata.m.color_encoding.WantICC()) return JXL_FAILURE("ICC unsupported");
    if (f->metadata.m.have_preview) return JXL_FAILURE("preview unsupported");
    JXL_RETURN_IF_ERROR(br.JumpToByteBoundary());
    return true;
  }();
  size_t hdr_bytes = br.TotalBitsConsumed() / kBitsPerByte;
  Status closed = br.Close();
  JXL_RETURN_IF_ERROR(ok);
  JXL_RETURN_IF_ERROR(closed);
  const uint8_t* frame_start = data + 2 + hdr_bytes;
  size_t frame_size = n - 2 - hdr_bytes;

  f->dec_state = jxl::make_unique<PassesDecoderState>(&f->mm);
  JXL_RETURN_IF_ERROR(f->dec_state->output_encoding_info.SetFromMetadata(f->metadata));
  // linear sRGB output, like djxl --color_space=RGB_D65_SRG_Rel_Lin
  JXL_RETURN_IF_ERROR(f->dec_state->output_encoding_info.MaybeSetColorEncoding(
      ColorEncoding::LinearSRGB(false)));
  f->decoded = jxl::make_unique<ImageBundle>(&f->mm, &f->metadata.m);

  FrameDecoder fd(f->dec_state.get(), f->metadata, f->pool.get(),
                  /*use_slow_rendering_pipeline=*/false);
  BitReader fr(Bytes(frame_start, frame_size));
  Status st = [&]() -> Status {
    JXL_RETURN_IF_ERROR(fd.InitFrame(&fr, f->decoded.get(), /*is_preview=*/false));
    JXL_RETURN_IF_ERROR(fd.InitFrameOutput());
    return true;
  }();
  size_t header_bytes = fr.TotalBitsConsumed() / kBitsPerByte;
  Status c2 = fr.Close();
  JXL_RETURN_IF_ERROR(st);
  JXL_RETURN_IF_ERROR(c2);
  f->frame_header = jxl::make_unique<FrameHeader>(&f->metadata);
  *f->frame_header = fd.GetFrameHeader();
  const FrameHeader& fh = *f->frame_header;
  if (fh.encoding != FrameEncoding::kVarDCT) return JXL_FAILURE("not VarDCT");
  if (!fh.chroma_subsampling.Is444()) return JXL_FAILURE("not 444");
  // (fh.upsampling != 1 is fine: UpsamplingStage, SURVEY.md §8f rank 4, follows the filters)
  if (fh.flags & (FrameHeader::kPatches | FrameHeader::kSplines))  // (kNoise: the noise stages follow the filters)
    return JXL_FAILURE("image features present");
  if (fh.passes.num_passes != 1) return JXL_FAILURE("multi-pass");
  const FrameDimensions fdim = fh.ToFrameDimensions();
  if (fdim.num_groups < 2) return JXL_FAILURE("single-section frame");

  Status close_ok = true;
  std::vector<std::unique_ptr<BitReader>> readers;
  std::vector<FrameDecoder::SectionInfo> early, late;
  {
    std::vector<std::unique_ptr<BitReaderScopedCloser>> closers;
    size_t pos = header_bytes;
    size_t index = 0;
    const size_t ac_global_id = fdim.num_dc_groups + 1;
    for (auto toc : fd.Toc()) {
      if (pos + toc.size > frame_size) return JXL_FAILURE("truncated");
      auto r = jxl::make_unique<BitReader>(Bytes(frame_start + pos, toc.size));
      FrameDecoder::SectionInfo si{r.get(), toc.id, index++};
      (toc.id <= ac_global_id ? early : late).push_back(si);
      closers.emplace_back(jxl::make_unique<BitReaderScopedCloser>(*r, close_ok));
      readers.emplace_back(std::move(r));
      pos += toc.size;
    }
    std::vector<FrameDecoder::SectionStatus> status(early.size());
    JXL_RETURN_IF_ERROR(fd.ProcessSections(early.data(), early.size(), status.data()));
    for (auto s : status) JXL_RETURN_IF_ERROR(s == FrameDecoder::kDone);
    // Switch on accumulate-mode storage: every group's coefficients land in
    // dec_state->coefficients->PlaneRow(c, group, offset).
    f->is16 = f->dec_state->coefficients->Type() == ACType::k16;
    if (f->storage == 1) {
      // the host-integration storage class (integration/pinned_ac_image.h) through libjxl's own
      // abstract ACImage interface: group-major [group][3][65536], malloc here, pinned in production
      if (f->is16) {
        auto im = jxlb_integration::GroupMajorACImage<int16_t>::Make(fdim.num_groups, malloc, free);
        if (!im) return JXL_FAILURE("alloc");
        f->raw_base = im->data();
        f->raw_bytes = im->size_bytes();
        f->dec_state->coefficients = std::move(im);
      } else {
        auto im = jxlb_integration::GroupMajorACImage<int32_t>::Make(fdim.num_groups, malloc, free);
        if (!im) return JXL_FAILURE("alloc");
        f->raw_base = im->data();
        f->raw_bytes = im->size_bytes();
        f->dec_state->coefficients = std::move(im);
      }
    } else if (f->is16) {
      JXL_ASSIGN_OR_RETURN(f->dec_state->coefficients,
                           ACImageT<int16_t>::Make(&f->mm, kGroupDim * kGroupDim,
                                                   fdim.num_groups));
    } else {
      JXL_ASSIGN_OR_RETURN(f->dec_state->coefficients,
                           ACImageT<int32_t>::Make(&f->mm, kGroupDim * kGroupDim,
                                                   fdim.num_groups));
    }
    f->dec_state->coefficients->ZeroFill();
    status.assign(late.size(), FrameDecoder::kSkipped);
    JXL_RETURN_IF_ERROR(fd.ProcessSections(late.data(), late.size(), status.data()));
    for (auto s : status) JXL_RETURN_IF_ERROR(s == FrameDecoder::kDone);
  }
  JXL_RETURN_IF_ERROR(close_ok);
  JXL_RETURN_IF_ERROR(fd.FinalizeFrame());
  // all 27 dequant matrices available to the exporter
  JXL_RETURN_IF_ERROR(f->dec_state->shared_storage.matrices.EnsureComputed(
      &f->mm, (1u << AcStrategy::kNumValidStrategies) - 1));

  // int32 copy for the roundtrip entry point
  JXL_ASSIGN_OR_RETURN(auto ac32, ACImageT<int32_t>::Make(&f->mm, kGroupDim * kGroupDim,
                                                         fdim.num_groups));
  for (size_t c = 0; c < 3; c++) {
    for (size_t g = 0; g < fdim.num_groups; g++) {
      int32_t* dst = ac32->PlaneRow(c, g, 0).ptr32;
      if (f->is16) {
        const int16_t* src = f->dec_state->coefficients->PlaneRow(c, g, 0).ptr16;
        for (size_t k = 0; k < kGroupDim * kGroupDim; k++) dst[k] = src[k];
      } else {
        memcpy(dst, f->dec_state->coefficients->PlaneRow(c, g, 0).ptr32,
               sizeof(int32_t) * kGroupDim * kGroupDim);
      }
    }
  }
  f->ac32.emplace_back(std::move(ac32));
  // Leave the decoder state in non-accumulate mode (empty k32 image) so that
  // DecodeGroupForRoundtrip reads only from `ac32` (dec_group.cc:219,343-355).
  f->stored = std::move(f->dec_state->coefficients);
  f->dec_state->coefficients = jxl::make_unique<ACImageT<int32_t>>();
  return true;
}

}  // namespace

struct RefFrameInfo {
  int32_t xsize, ysize, xsize_blocks, ysize_blocks;
  int32_t xsize_groups, ysize_groups, num_groups, ac_is16;
  int32_t cmap_xsize, cmap_ysize;           // 64x64-px tiles
  int32_t gab, epf_iters;
  float inv_global_scale, global_scale_float;  // Quantizer::InvGlobalScale / Scale
  float x_dm_multiplier, b_dm_multiplier;
  float quant_biases[4];
  float cfl_base_x, cfl_base_b, cfl_color_scale;  // YtoXRatio = base + f*scale
  float gab_weights[6];                     // x1 x2 y1 y2 b1 b2
  float epf_sharp_lut[8];
  float epf_channel_scale[3];
  float epf_quant_mul, epf_pass0_sigma_scale, epf_pass2_sigma_scale, epf_border_sad_mul;
  float inverse_opsin_matrix[9];            // already x 255/intensity_target
  float opsin_biases[4];                    // "neg_bias" (3 used)
  float opsin_biases_cbrt[4];
  int32_t dequant_table_floats;             // 2056*64*3
  int32_t dequant_offsets[27 * 3];          // float offset of Matrix(kind,c)
  int32_t upsampling;                       // frame_header.upsampling (1, 2, 4, 8)
  int32_t xsize_upsampled, ysize_upsampled; // FrameDimensions (frame_dimensions.h:34-60)
  float upsampling_weights[210];            // CustomTransformData::upsampling{2,4,8}_weights of that factor (15 / 55 / 210 used)
  int32_t ycbcr;                            // frame_header.color_transform == kYCbCr (JPEG-origin frames)
  int32_t noise;                            // frame_header.flags & kNoise
  float noise_lut[8];                       // NoiseParams::lut (noise.h:27-43)
  uint32_t visible_frame_index, nonvisible_frame_index;  // PassesDecoderState, seeds of the noise generator
};

REF_API void* ref_frame_open_storage(const uint8_t* jxl, size_t n, int threads, int storage);
REF_API void* ref_frame_open(const uint8_t* jxl, size_t n, int threads) {
  return ref_frame_open_storage(jxl, n, threads, 0);
}

// The libjxl-side binding of the product ABI (integration/gpu_frame_binding.h) applied to this frame's
// live decoder state: *out points into the reference's own images (valid until ref_frame_close).
REF_API int ref_frame_bind_gpu_frame(void* h, uint32_t out_format, uint32_t stage_mask, jxlgpu_frame* out) {
  auto* f = static_cast<RefFrame*>(h);
  if (!jxlb_integration::IsEligible(*f->frame_header, f->metadata)) return 2;
  if (!jxlb_integration::BindGpuFrame(*f->dec_state, *f->frame_header, out_format, stage_mask, &f->binding)) return 1;
  // this harness parked the coefficient image elsewhere after decoding (OpenImpl), so the type the
  // binding read from dec_state->coefficients is the placeholder's: restore the frame's own
  f->binding.frame.ac_type = f->is16 ? JXLGPU_AC_INT16 : JXLGPU_AC_INT32;
  *out = f->binding.frame;
  return 0;
}

// the raw group-major coefficient allocation of a frame opened with storage == 1
REF_API int ref_frame_raw_coeffs(void* h, void** base, size_t* bytes) {
  auto* f = static_cast<RefFrame*>(h);
  if (!f->raw_base) return 1;
  *base = f->raw_base;
  *bytes = f->raw_bytes;
  return 0;
}

REF_API void* ref_frame_open_storage(const uint8_t* jxl, size_t n, int threads, int storage) {
  auto* f = new RefFrame();
  f->storage = storage;
  f->runner = JxlThreadParallelRunnerCreate(nullptr, threads < 1 ? 1 : threads);
  f->pool.reset(new ThreadPool(JxlThreadParallelRunner, f->runner));
  Status st = OpenImpl(f, jxl, n);
  if (!st) {
    delete f;
    return nullptr;
  }
  return f;
}
REF_API void ref_frame_close(void* h) { delete static_cast<RefFrame*>(h); }

REF_API int ref_frame_info(void* h, RefFrameInfo* o) {
  auto* f = static_cast<RefFrame*>(h);
  const PassesSharedState& sh = *f->dec_state->shared;
  const FrameDimensions& d = sh.frame_dim;
  const LoopFilter& lf = f->frame_header->loop_filter;
  memset(o, 0, sizeof(*o));
  o->xsize = d.xsize; o->ysize = d.ysize;
  o->xsize_blocks = d.xsize_blocks; o->ysize_blocks = d.ysize_blocks;
  o->xsize_groups = d.xsize_groups; o->ysize_groups = d.ysize_groups;
  o->num_groups = d.num_groups; o->ac_is16 = f->is16;
  o->cmap_xsize = sh.cmap.ytox_map.xsize(); o->cmap_ysize = sh.cmap.ytox_map.ysize();
  o->gab = lf.gab; o->epf_iters = lf.epf_iters;
  o->inv_global_scale = sh.quantizer.InvGlobalScale();
  o->global_scale_float = sh.quantizer.Scale();
  o->x_dm_multiplier = f->dec_state->x_dm_multiplier;
  o->b_dm_multiplier = f->dec_state->b_dm_multiplier;
  const OpsinParams& op = f->dec_state->output_encoding_info.opsin_params;
  memcpy(o->quant_biases, op.quant_biases, sizeof(o->quant_biases));
  const ColorCorrelation& cc = sh.cmap.base();
  o->cfl_base_x = cc.GetBaseCorrelationX();
  o->cfl_base_b = cc.GetBaseCorrelationB();
  o->cfl_color_scale = cc.YtoXRatio(1) - cc.YtoXRatio(0);
  // exact color_scale_: 1.0f / color_factor_ (chroma_from_luma.h:77-79)
  o->cfl_color_scale = 1.0f / static_cast<uint32_t>(cc.GetColorFactor());
  o->gab_weights[0] = lf.gab_x_weight1; o->gab_weights[1] = lf.gab_x_weight2;
  o->gab_weights[2] = lf.gab_y_weight1; o->gab_weights[3] = lf.gab_y_weight2;
  o->gab_weights[4] = lf.gab_b_weight1; o->gab_weights[5] = lf.gab_b_weight2;
  memcpy(o->epf_sharp_lut, lf.epf_sharp_lut, sizeof(o->epf_sharp_lut));
  memcpy(o->epf_channel_scale, lf.epf_channel_scale, sizeof(o->epf_channel_scale));
  o->epf_quant_mul = lf.epf_quant_mul;
  o->epf_pass0_sigma_scale = lf.epf_pass0_sigma_scale;
  o->epf_pass2_sigma_scale = lf.epf_pass2_sigma_scale;
  o->epf_border_sad_mul = lf.epf_border_sad_mul;
  for (int i = 0; i < 9; i++) o->inverse_opsin_matrix[i] = op.inverse_opsin_matrix[i * 4];
  memcpy(o->opsin_biases, op.opsin_biases, sizeof(o->opsin_biases));
  memcpy(o->opsin_biases_cbrt, op.opsin_biases_cbrt, sizeof(o->opsin_biases_cbrt));
  const float* base = sh.matrices.Matrix(AcStrategyType::DCT, 0);
  for (int k = 0; k < 27; k++)
    for (int c = 0; c < 3; c++) {
      const float* p = sh.matrices.Matrix(static_cast<AcStrategyType>(k), c);
      if (p < base) base = p;
    }
  o->upsampling = static_cast<int32_t>(f->frame_header->upsampling);
  o->xsize_upsampled = d.xsize_upsampled;
  o->ysize_upsampled = d.ysize_upsampled;
  {
    const CustomTransformData& td = f->frame_header->nonserialized_metadata->transform_data;
    const float* w = o->upsampling == 2 ? td.upsampling2_weights : o->upsampling == 4 ? td.upsampling4_weights : td.upsampling8_weights;
    const size_t n = o->upsampling == 2 ? 15 : o->upsampling == 4 ? 55 : 210;
    memcpy(o->upsampling_weights, w, n * sizeof(float));
  }
  o->ycbcr = f->frame_header->color_transform == ColorTransform::kYCbCr ? 1 : 0;
  o->noise = (f->frame_header->flags & FrameHeader::kNoise) ? 1 : 0;
  for (int i = 0; i < 8; i++) o->noise_lut[i] = sh.image_features.noise_params.lut[i];
  o->visible_frame_index = static_cast<uint32_t>(f->dec_state->visible_frame_index);
  o->nonvisible_frame_index = static_cast<uint32_t>(f->dec_state->nonvisible_frame_index);
  o->dequant_table_floats = DequantMatrices::kSumRequiredXy * kDCTBlockSize * 3;
  for (int k = 0; k < 27; k++)
    for (int c = 0; c < 3; c++)
      o->dequant_offsets[k * 3 + c] =
          sh.matrices.Matrix(static_cast<AcStrategyType>(k), c) - base;
  return 0;
}

// ---------------------------------------------------------------------------
// (3b) override the frame-header / image-metadata parameters of an opened frame,
// as if the bitstream had carried them: the LoopFilter's custom Gaborish / EPF
// fields, the qm-scale dequantisation multipliers, the DC colour-correlation
// header (base correlations, colour factor) and the metadata's opsin inverse
// matrix (already x 255 / intensity_target), opsin and quantisation biases.
// The sigma image is recomputed with the reference's ComputeSigma, because the
// EPF fields feed it.  Values must be ones the bitstream can carry: the base
// correlations go through the reference's own F16 decoder.
// ---------------------------------------------------------------------------
struct RefFrameParams {
  float x_dm_multiplier, b_dm_multiplier;
  float quant_biases[4];
  float cfl_base_x, cfl_base_b;
  uint32_t color_factor;
  float gab_weights[6];                     // x1 x2 y1 y2 b1 b2
  float epf_sharp_lut[8];
  float epf_channel_scale[3];
  float epf_quant_mul, epf_pass0_sigma_scale, epf_pass2_sigma_scale, epf_border_sad_mul;
  float inverse_opsin_matrix[9];
  float opsin_biases[3];
};

namespace {

// LSB-first bit packing, the order BitReader reads in
struct BitPacker {
  std::vector<uint8_t> bytes = std::vector<uint8_t>(32, 0);
  size_t pos = 0;
  void Put(uint32_t v, size_t n) {
    for (size_t i = 0; i < n; i++, pos++)
      if ((v >> i) & 1) bytes[pos / 8] |= static_cast<uint8_t>(1u << (pos % 8));
  }
};

// IEEE binary16 bits of f; false when f is not exactly representable (no inf / NaN in F16 fields)
bool HalfBits(float f, uint32_t* bits) {
  const uint32_t sign = std::signbit(f) ? 0x8000u : 0u;
  const float a = std::fabs(f);
  if (a == 0.0f) { *bits = sign; return true; }
  int e;
  std::frexp(a, &e);                        // a = m * 2^e, m in [0.5, 1)
  const int biased = e - 1 + 15;
  if (biased > 30) return false;
  const float unit = std::ldexp(1.0f, (biased >= 1 ? e - 1 : -14) - 10);   // value of one mantissa step
  const float steps = a / unit;
  const uint32_t m = static_cast<uint32_t>(steps);
  if (static_cast<float>(m) != steps) return false;
  *bits = biased >= 1 ? sign | (static_cast<uint32_t>(biased) << 10) | (m - 1024) : sign | m;
  return true;
}

Status SetParamsImpl(RefFrame* f, const RefFrameParams& p) {
  LoopFilter& lf = f->frame_header->loop_filter;
  lf.gab_custom = true;
  lf.gab_x_weight1 = p.gab_weights[0]; lf.gab_x_weight2 = p.gab_weights[1];
  lf.gab_y_weight1 = p.gab_weights[2]; lf.gab_y_weight2 = p.gab_weights[3];
  lf.gab_b_weight1 = p.gab_weights[4]; lf.gab_b_weight2 = p.gab_weights[5];
  lf.epf_sharp_custom = true;
  memcpy(lf.epf_sharp_lut, p.epf_sharp_lut, sizeof(lf.epf_sharp_lut));
  lf.epf_weight_custom = true;
  memcpy(lf.epf_channel_scale, p.epf_channel_scale, sizeof(lf.epf_channel_scale));
  lf.epf_sigma_custom = true;
  lf.epf_quant_mul = p.epf_quant_mul;
  lf.epf_pass0_sigma_scale = p.epf_pass0_sigma_scale;
  lf.epf_pass2_sigma_scale = p.epf_pass2_sigma_scale;
  lf.epf_border_sad_mul = p.epf_border_sad_mul;

  PassesDecoderState* ds = f->dec_state.get();
  ds->x_dm_multiplier = p.x_dm_multiplier;
  ds->b_dm_multiplier = p.b_dm_multiplier;
  OpsinParams& op = ds->output_encoding_info.opsin_params;
  for (int i = 0; i < 9; i++)
    for (int lane = 0; lane < 4; lane++) op.inverse_opsin_matrix[i * 4 + lane] = p.inverse_opsin_matrix[i];
  for (int c = 0; c < 3; c++) {
    op.opsin_biases[c] = p.opsin_biases[c];
    op.opsin_biases_cbrt[c] = cbrtf(p.opsin_biases[c]);
  }
  memcpy(op.quant_biases, p.quant_biases, sizeof(op.quant_biases));

  // the DC colour-correlation header: not all default, colour factor (U32), two F16 base correlations, and
  // the frame's own DC correlations again (RecomputeDCFactors keeps them)
  ColorCorrelationMap& cmap = ds->shared_storage.cmap;
  const ColorCorrelation& cc = cmap.base();
  BitPacker bits;
  bits.Put(0, 1);
  const uint32_t cf = p.color_factor;
  if (cf == kDefaultColorFactor) bits.Put(0, 2);
  else if (cf == 256) bits.Put(1, 2);
  else if (cf >= 2 && cf < 258) { bits.Put(2, 2); bits.Put(cf - 2, 8); }
  else if (cf >= 258 && cf < 258 + 65536) { bits.Put(3, 2); bits.Put(cf - 258, 16); }
  else return JXL_FAILURE("colour factor out of range");
  uint32_t hx, hb;
  if (!HalfBits(p.cfl_base_x, &hx) || !HalfBits(p.cfl_base_b, &hb)) return JXL_FAILURE("base correlation not F16");
  bits.Put(hx, 16);
  bits.Put(hb, 16);
  bits.Put(static_cast<uint32_t>(cc.GetYToXDC() - std::numeric_limits<int8_t>::min()), 8);
  bits.Put(static_cast<uint32_t>(cc.GetYToBDC() - std::numeric_limits<int8_t>::min()), 8);
  {
    BitReader br(Bytes(bits.bytes.data(), bits.bytes.size()));
    Status st = cmap.DecodeDC(&br);
    Status closed = br.Close();
    JXL_RETURN_IF_ERROR(st);
    JXL_RETURN_IF_ERROR(closed);
  }
  if (cmap.base().GetBaseCorrelationX() != p.cfl_base_x || cmap.base().GetBaseCorrelationB() != p.cfl_base_b ||
      static_cast<uint32_t>(cmap.base().GetColorFactor()) != cf)
    return JXL_FAILURE("colour correlation not taken");

  if (lf.epf_iters > 0) {   // as the DC groups do after their AC metadata (dec_modular.cc:557-559)
    const FrameDimensions& d = ds->shared->frame_dim;
    for (size_t g = 0; g < d.num_dc_groups; g++) JXL_RETURN_IF_ERROR(ComputeSigma(lf, d.DCGroupRect(g), ds));
  }
  return true;
}

}  // namespace

REF_API int ref_frame_set_params(void* h, const RefFrameParams* p) {
  return SetParamsImpl(static_cast<RefFrame*>(h), *p) ? 0 : 1;
}

// (3c) custom upsampling weights of factor N (2, 4, 8: 15 / 55 / 210 values) as if the image header had carried
// them: the metadata's CustomTransformData with that bit of custom_weights_mask set, written with the reference's
// own Bundle writer and read back with Bundle::Read into the frame's transform_data, which UpsamplingStage and
// ref_frame_info read.  Every value must be exactly F16.
namespace {
Status SetUpsamplingWeightsImpl(RefFrame* f, int n, const float* w) {
  const size_t count = n == 2 ? 15 : n == 4 ? 55 : n == 8 ? 210 : 0;
  if (!count) return JXL_FAILURE("upsampling factor");
  for (size_t i = 0; i < count; i++) {
    uint32_t bits;
    if (!HalfBits(w[i], &bits)) return JXL_FAILURE("upsampling weight not F16");
  }
  CustomTransformData td = f->metadata.transform_data;
  td.nonserialized_xyb_encoded = f->metadata.m.xyb_encoded;
  const uint32_t bit = n == 2 ? 1u : n == 4 ? 2u : 4u;
  td.custom_weights_mask |= bit;
  float* dst = n == 2 ? td.upsampling2_weights : n == 4 ? td.upsampling4_weights : td.upsampling8_weights;
  memcpy(dst, w, count * sizeof(float));
  BitWriter writer(&f->mm);
  JXL_RETURN_IF_ERROR(Bundle::Write(td, &writer, LayerType::Header, nullptr));
  writer.ZeroPadToByte();
  const Span<const uint8_t> span = writer.GetSpan();
  CustomTransformData back;
  back.nonserialized_xyb_encoded = td.nonserialized_xyb_encoded;
  BitReader br(Bytes(span.data(), span.size()));
  Status st = Bundle::Read(&br, &back);
  Status closed = br.Close();
  JXL_RETURN_IF_ERROR(st);
  JXL_RETURN_IF_ERROR(closed);
  const float* got = n == 2 ? back.upsampling2_weights : n == 4 ? back.upsampling4_weights : back.upsampling8_weights;
  if (!(back.custom_weights_mask & bit) || memcmp(got, w, count * sizeof(float)))
    return JXL_FAILURE("upsampling weights not taken");
  f->metadata.transform_data = back;
  return true;
}

// (3d) the noise strength LUT as the frame header's noise parameters carry it: eight 10-bit codes read by the
// reference's DecodeNoise (lut[i] = code / 1024).  Every value must be k / 1024 with k <= 1023.
Status SetNoiseLutImpl(RefFrame* f, const float* lut) {
  BitPacker bits;
  for (int i = 0; i < 8; i++) {
    const float k = lut[i] * 1024.0f;
    if (!(k >= 0.0f && k <= 1023.0f) || k != std::floor(k)) return JXL_FAILURE("noise LUT entry not k / 1024");
    bits.Put(static_cast<uint32_t>(k), 10);
  }
  NoiseParams np;
  BitReader br(Bytes(bits.bytes.data(), bits.bytes.size()));
  Status st = DecodeNoise(&br, &np);
  Status closed = br.Close();
  JXL_RETURN_IF_ERROR(st);
  JXL_RETURN_IF_ERROR(closed);
  for (int i = 0; i < 8; i++)
    if (np.lut[i] != lut[i]) return JXL_FAILURE("noise LUT not taken");
  f->dec_state->shared_storage.image_features.noise_params = np;
  return true;
}
}  // namespace

REF_API int ref_frame_set_upsampling_weights(void* h, int n, const float* w) {
  return SetUpsamplingWeightsImpl(static_cast<RefFrame*>(h), n, w) ? 0 : 1;
}

// (the frame must carry the noise flag: the encoder's photon noise sets it)
REF_API int ref_frame_set_noise_lut(void* h, const float* lut) {
  auto* f = static_cast<RefFrame*>(h);
  if (!(f->frame_header->flags & FrameHeader::kNoise)) return 2;
  return SetNoiseLutImpl(f, lut) ? 0 : 1;
}

// plane ids for ref_frame_get_plane
enum {
  REF_PLANE_AC_STRATEGY = 0,  // u8  [ysize_blocks][xsize_blocks]  (type<<1)|first
  REF_PLANE_RAW_QUANT = 1,    // i32 [ysize_blocks][xsize_blocks]
  REF_PLANE_SHARPNESS = 2,    // u8  [ysize_blocks][xsize_blocks]
  REF_PLANE_YTOX = 3,         // i8  [cmap_ysize][cmap_xsize]
  REF_PLANE_YTOB = 4,         // i8
  REF_PLANE_DC = 5,           // f32 [3][ysize_blocks][xsize_blocks]
  REF_PLANE_SIGMA = 6,        // f32 [ysize_blocks+4][xsize_blocks+4] (inv sigma)
  REF_PLANE_DEQUANT = 7,      // f32 [dequant_table_floats]
  REF_PLANE_COEFFS = 8,       // i16|i32 [3][num_groups][65536]
  REF_PLANE_DECODED = 9,      // f32 [ysize][xsize][3] reference decode (linear sRGB)
};

REF_API int ref_frame_get_plane(void* h, int which, void* out, size_t out_bytes) {
  auto* f = static_cast<RefFrame*>(h);
  const PassesSharedState& sh = *f->dec_state->shared;
  const FrameDimensions& d = sh.frame_dim;
  const size_t xb = d.xsize_blocks, yb = d.ysize_blocks;
  auto need = [&](size_t b) { return b <= out_bytes; };
  switch (which) {
    case REF_PLANE_AC_STRATEGY: {
      if (!need(xb * yb)) return 2;
      uint8_t* o = static_cast<uint8_t*>(out);
      for (size_t y = 0; y < yb; y++) {
        AcStrategyRow row = sh.ac_strategy.ConstRow(y);
        for (size_t x = 0; x < xb; x++) {
          AcStrategy a = row[x];
          o[y * xb + x] = (a.RawStrategy() << 1) | (a.IsFirstBlock() ? 1 : 0);
        }
      }
      return 0;
    }
    case REF_PLANE_RAW_QUANT: {
      if (!need(xb * yb * 4)) return 2;
      for (size_t y = 0; y < yb; y++)
        memcpy(static_cast<int32_t*>(out) + y * xb, sh.raw_quant_field.ConstRow(y), xb * 4);
      return 0;
    }
    case REF_PLANE_SHARPNESS: {
      if (!need(xb * yb)) return 2;
      for (size_t y = 0; y < yb; y++)
        memcpy(static_cast<uint8_t*>(out) + y * xb, sh.epf_sharpness.ConstRow(y), xb);
      return 0;
    }
    case REF_PLANE_YTOX:
    case REF_PLANE_YTOB: {
      const ImageSB& m = which == REF_PLANE_YTOX ? sh.cmap.ytox_map : sh.cmap.ytob_map;
      if (!need(m.xsize() * m.ysize())) return 2;
      for (size_t y = 0; y < m.ysize(); y++)
        memcpy(static_cast<int8_t*>(out) + y * m.xsize(), m.ConstRow(y), m.xsize());
      return 0;
    }
    case REF_PLANE_DC: {
      if (!need(3 * xb * yb * 4)) return 2;
      for (size_t c = 0; c < 3; c++)
        for (size_t y = 0; y < yb; y++)
          memcpy(static_cast<float*>(out) + (c * yb + y) * xb, sh.dc->ConstPlaneRow(c, y),
                 xb * 4);
      return 0;
    }
    case REF_PLANE_SIGMA: {
      const ImageF& s = f->dec_state->sigma;
      if (s.xsize() == 0) return 3;
      if (!need((xb + 4) * (yb + 4) * 4)) return 2;
      for (size_t y = 0; y < yb + 4; y++)
        memcpy(static_cast<float*>(out) + y * (xb + 4), s.ConstRow(y), (xb + 4) * 4);
      return 0;
    }
    case REF_PLANE_DEQUANT: {
      RefFrameInfo info;
      ref_frame_info(h, &info);
      if (!need(static_cast<size_t>(info.dequant_table_floats) * 4)) return 2;
      const float* base = sh.matrices.Matrix(AcStrategyType::DCT, 0) - info.dequant_offsets[0];
      memcpy(out, base, static_cast<size_t>(info.dequant_table_floats) * 4);
      return 0;
    }
    case REF_PLANE_COEFFS: {
      const size_t per = kGroupDim * kGroupDim;
      const size_t es = f->is16 ? 2 : 4;
      if (!need(3 * d.num_groups * per * es)) return 2;
      for (size_t c = 0; c < 3; c++)
        for (size_t g = 0; g < d.num_groups; g++) {
          uint8_t* dst = static_cast<uint8_t*>(out) + (c * d.num_groups + g) * per * es;
          if (f->is16) memcpy(dst, f->stored->PlaneRow(c, g, 0).ptr16, per * es);
          else memcpy(dst, f->stored->PlaneRow(c, g, 0).ptr32, per * es);
        }
      return 0;
    }
    case REF_PLANE_DECODED: {
      const size_t dx = d.xsize_upsampled, dy = d.ysize_upsampled;  // (== xsize, ysize without upsampling)
      if (!need(dx * dy * 3 * 4)) return 2;
      const Image3F& img = *f->decoded->color();
      float* o = static_cast<float*>(out);
      for (size_t y = 0; y < dy; y++)
        for (size_t c = 0; c < 3; c++) {
          const float* r = img.ConstPlaneRow(c, y);
          for (size_t x = 0; x < dx; x++) o[(y * dx + x) * 3 + c] = r[x];
        }
      return 0;
    }
  }
  return 1;
}

// ---------------------------------------------------------------------------
// (4) hot path only, from the retained coefficients, with the reference's own
// code: DecodeGroupForRoundtrip (lib/jxl/dec_group.cc:820-841) feeding a
// pipeline made of the requested subset of the reference stages.  Loop
// structure follows RoundtripImage (lib/jxl/enc_adaptive_quantization.cc:840-915).
// stage_mask bits: 1 gab, 2 epf0, 4 epf1, 8 epf2, 16 xyb->linear.  -1 = the
// frame's own chain (gab/epf per its LoopFilter) + xyb.
// out: planar f32 [3][ysize][xsize] (may be NULL when only timing).
// reps: number of timed repetitions; seconds[] gets each repetition's time.
// ---------------------------------------------------------------------------
REF_API int ref_frame_render(void* h, int stage_mask, float* out, int reps, double* seconds) {
  auto* f = static_cast<RefFrame*>(h);
  PassesDecoderState* ds = f->dec_state.get();
  const FrameHeader& fh = *f->frame_header;
  const LoopFilter& lf = fh.loop_filter;
  const FrameDimensions& d = ds->shared->frame_dim;
  if (stage_mask < 0) {
    stage_mask = 16 | (lf.gab ? 1 : 0);
    if (lf.epf_iters >= 3) stage_mask |= 2;
    if (lf.epf_iters >= 1) stage_mask |= 4;
    if (lf.epf_iters >= 2) stage_mask |= 8;
  }
  if ((stage_mask & 14) && lf.epf_iters == 0) return 7;  // no sigma image
  if (reps < 1) reps = 1;
  const bool with_noise = (stage_mask & 128) && (fh.flags & FrameHeader::kNoise);
  // The pipeline, the per-thread scratch and the output image are set up once and reused by
  // every timed repetition (ClearDone() re-arms the groups, as progressive passes do,
  // dec_frame.cc:700-705): the timed region is the hot path only, no allocation, no page faults.
  Image3F result;
  AlignedArray<GroupDecCache> caches;
  size_t caches_n = 0;
  const auto init = [&](size_t num_threads) -> Status {
    if (caches_n >= num_threads) return true;
    caches_n = num_threads;
    JXL_RETURN_IF_ERROR(ds->render_pipeline->PrepareForThreads(num_threads, false));
    JXL_ASSIGN_OR_RETURN(caches, AlignedArray<GroupDecCache>::Create(&f->mm, num_threads));
    return true;
  };
  const auto group = [&](uint32_t g, size_t thread) -> Status {
    RenderPipelineInput input = ds->render_pipeline->GetInputBuffers(g, thread);
    JXL_RETURN_IF_ERROR(DecodeGroupForRoundtrip(fh, f->ac32, g, ds, &caches[thread], thread, input,
                                                nullptr, nullptr));
    if (with_noise) PrepareNoiseInput(*ds, d, fh, g, thread);  // as ProcessACGroup does (dec_frame.cc:545-548)
    JXL_RETURN_IF_ERROR(input.Done());
    return true;
  };
  Status st = [&]() -> Status {
    RenderPipeline::Builder builder(&f->mm, with_noise ? 6 : 3);
    if (stage_mask & 1) JXL_RETURN_IF_ERROR(builder.AddStage(GetGaborishStage(lf)));
    if (stage_mask & 2)
      JXL_RETURN_IF_ERROR(builder.AddStage(GetEPFStage(lf, ds->sigma, EpfStage::Zero)));
    if (stage_mask & 4)
      JXL_RETURN_IF_ERROR(builder.AddStage(GetEPFStage(lf, ds->sigma, EpfStage::One)));
    if (stage_mask & 8)
      JXL_RETURN_IF_ERROR(builder.AddStage(GetEPFStage(lf, ds->sigma, EpfStage::Two)));
    if ((stage_mask & 64) && fh.upsampling != 1) {  // UpsamplingStage per colour channel, where PreparePipeline puts it (dec_cache.cc:216-227)
      for (size_t c = 0; c < 3; c++)
        JXL_RETURN_IF_ERROR(builder.AddStage(GetUpsamplingStage(&f->mm, fh.nonserialized_metadata->transform_data, c,
                                                                CeilLog2Nonzero(fh.upsampling))));
    }
    if (with_noise) {  // ConvolveNoise + AddNoise on three extra channels (dec_cache.cc:232-236)
      JXL_RETURN_IF_ERROR(builder.AddStage(GetConvolveNoiseStage(3)));
      JXL_RETURN_IF_ERROR(builder.AddStage(GetAddNoiseStage(ds->shared->image_features.noise_params,
                                                            ds->shared->cmap.base(), 3)));
    }
    if (stage_mask & 16) {  // the frame's colour transform (dec_cache.cc:259-267)
      if (fh.color_transform == ColorTransform::kYCbCr) JXL_RETURN_IF_ERROR(builder.AddStage(GetYCbCrStage()));
      else JXL_RETURN_IF_ERROR(builder.AddStage(GetXYBStage(ds->output_encoding_info)));
    }
    JXL_RETURN_IF_ERROR(builder.AddStage(GetWriteToImage3FStage(&f->mm, &result)));
    JXL_ASSIGN_OR_RETURN(ds->render_pipeline, std::move(builder).Finalize(d));
    // warm-up pass (untimed): allocates and touches everything
    JXL_RETURN_IF_ERROR(RunOnPool(f->pool.get(), 0, d.num_groups, init, group, "hot path"));
    return true;
  }();
  if (!st) return 1;
  const bool ups = (stage_mask & 64) && fh.upsampling != 1;
  const size_t ox = ups ? d.xsize_upsampled : d.xsize, oy = ups ? d.ysize_upsampled : d.ysize;
  if (out) {
    if (result.xsize() != ox || result.ysize() != oy) return 5;
    for (size_t c = 0; c < 3; c++)
      for (size_t y = 0; y < oy; y++)
        memcpy(out + (c * oy + y) * ox, result.ConstPlaneRow(c, y), ox * sizeof(float));
  }
  for (int rep = 0; rep < reps; rep++) {
    for (size_t g = 0; g < d.num_groups; g++) ds->render_pipeline->ClearDone(g);
    double t0 = NowSec();
    Status s2 = RunOnPool(f->pool.get(), 0, d.num_groups, init, group, "hot path");
    double t1 = NowSec();
    if (!s2) return 1;
    if (seconds) seconds[rep] = t1 - t0;
  }
  if (out && getenv("REF_CHECK_RERUN")) {  // the re-armed passes produce the same pixels
    for (size_t c = 0; c < 3; c++)
      for (size_t y = 0; y < oy; y++)
        if (memcmp(out + (c * oy + y) * ox, result.ConstPlaneRow(c, y), ox * sizeof(float)))
          return 9;
  }
  return 0;
}

// ---------------------------------------------------------------------------
// (4b) same loop, but ending the way the decoder's real pipeline ends
// (dec_cache.cc:259-330): optional FromLinearStage with an sRGB output encoding
// (stage_mask bit 32, stage_from_linear.cc:161-166) and WriteToOutputStage
// into a caller buffer of a JxlPixelFormat (stage_write.cc:455-700).
// out_format: 0 = {3, FLOAT}, 2 = {3, UINT8}, 3 = {4, UINT8}, 4 = {3, UINT16},
// 5 = {3, FLOAT16}; native endianness, dense rows.  out may be NULL (timing).
// ---------------------------------------------------------------------------
REF_API int ref_frame_render_out(void* h, int stage_mask, int out_format, void* out, int reps,
                                 double* seconds) {
  auto* f = static_cast<RefFrame*>(h);
  PassesDecoderState* ds = f->dec_state.get();
  const FrameHeader& fh = *f->frame_header;
  const LoopFilter& lf = fh.loop_filter;
  const FrameDimensions& d = ds->shared->frame_dim;
  if (stage_mask < 0) {
    const int srgb = (-stage_mask) & 32 ? 32 : 0;  // -1: derived chain; -33: derived chain + sRGB
    stage_mask = 16 | srgb | (lf.gab ? 1 : 0);
    if (lf.epf_iters >= 3) stage_mask |= 2;
    if (lf.epf_iters >= 1) stage_mask |= 4;
    if (lf.epf_iters >= 2) stage_mask |= 8;
  }
  if ((stage_mask & 14) && lf.epf_iters == 0) return 7;
  if (reps < 1) reps = 1;
  JxlPixelFormat format = {3, JXL_TYPE_FLOAT, JXL_NATIVE_ENDIAN, 0};
  size_t bits = 32, px_bytes = 12;
  switch (out_format) {
    case 0: break;
    case 2: format = {3, JXL_TYPE_UINT8, JXL_NATIVE_ENDIAN, 0}; bits = 8; px_bytes = 3; break;
    case 3: format = {4, JXL_TYPE_UINT8, JXL_NATIVE_ENDIAN, 0}; bits = 8; px_bytes = 4; break;
    case 4: format = {3, JXL_TYPE_UINT16, JXL_NATIVE_ENDIAN, 0}; bits = 16; px_bytes = 6; break;
    case 5: format = {3, JXL_TYPE_FLOAT16, JXL_NATIVE_ENDIAN, 0}; bits = 16; px_bytes = 6; break;
    default: return 8;
  }
  std::vector<uint8_t> own;
  const size_t stride = d.xsize * px_bytes;
  if (!out) {
    own.resize(stride * d.ysize);
    out = own.data();
  }
  ImageOutput main_output = {};
  main_output.format = format;
  main_output.bits_per_sample = bits;
  main_output.buffer = out;
  main_output.buffer_size = stride * d.ysize;
  main_output.stride = stride;
  std::vector<ImageOutput> extra;
  AlignedArray<GroupDecCache> caches;
  size_t caches_n = 0;
  const auto init = [&](size_t num_threads) -> Status {
    if (caches_n >= num_threads) return true;
    caches_n = num_threads;
    JXL_RETURN_IF_ERROR(ds->render_pipeline->PrepareForThreads(num_threads, false));
    JXL_ASSIGN_OR_RETURN(caches, AlignedArray<GroupDecCache>::Create(&f->mm, num_threads));
    return true;
  };
  const auto group = [&](uint32_t g, size_t thread) -> Status {
    RenderPipelineInput input = ds->render_pipeline->GetInputBuffers(g, thread);
    JXL_RETURN_IF_ERROR(DecodeGroupForRoundtrip(fh, f->ac32, g, ds, &caches[thread], thread, input,
                                                nullptr, nullptr));
    JXL_RETURN_IF_ERROR(input.Done());
    return true;
  };
  Status st = [&]() -> Status {
    RenderPipeline::Builder builder(&f->mm, 3);
    if (stage_mask & 1) JXL_RETURN_IF_ERROR(builder.AddStage(GetGaborishStage(lf)));
    if (stage_mask & 2)
      JXL_RETURN_IF_ERROR(builder.AddStage(GetEPFStage(lf, ds->sigma, EpfStage::Zero)));
    if (stage_mask & 4)
      JXL_RETURN_IF_ERROR(builder.AddStage(GetEPFStage(lf, ds->sigma, EpfStage::One)));
    if (stage_mask & 8)
      JXL_RETURN_IF_ERROR(builder.AddStage(GetEPFStage(lf, ds->sigma, EpfStage::Two)));
    if (stage_mask & 16) {  // the frame's colour transform (dec_cache.cc:259-267)
      if (fh.color_transform == ColorTransform::kYCbCr) JXL_RETURN_IF_ERROR(builder.AddStage(GetYCbCrStage()));
      else JXL_RETURN_IF_ERROR(builder.AddStage(GetXYBStage(ds->output_encoding_info)));
    }
    if (stage_mask & 32) {
      OutputEncodingInfo info = ds->output_encoding_info;
      info.color_encoding = ColorEncoding::SRGB(/*is_gray=*/false);
      JXL_RETURN_IF_ERROR(builder.AddStage(GetFromLinearStage(info)));
    }
    JXL_RETURN_IF_ERROR(builder.AddStage(GetWriteToOutputStage(main_output, d.xsize, d.ysize,
                                                               /*has_alpha=*/false, /*unpremul_alpha=*/false,
                                                               /*alpha_c=*/0, Orientation::kIdentity, extra,
                                                               &f->mm)));
    JXL_ASSIGN_OR_RETURN(ds->render_pipeline, std::move(builder).Finalize(d));
    JXL_RETURN_IF_ERROR(RunOnPool(f->pool.get(), 0, d.num_groups, init, group, "hot path"));
    return true;
  }();
  if (!st) return 1;
  for (int rep = 0; rep < reps; rep++) {
    for (size_t g = 0; g < d.num_groups; g++) ds->render_pipeline->ClearDone(g);
    double t0 = NowSec();
    Status s2 = RunOnPool(f->pool.get(), 0, d.num_groups, init, group, "hot path");
    double t1 = NowSec();
    if (!s2) return 1;
    if (seconds) seconds[rep] = t1 - t0;
  }
  return 0;
}

// ---------------------------------------------------------------------------
// (5) function-level facade (lib/jxl/dec_transforms_testonly.h:20-30), the
// same entry points ac_strategy_test.cc drives for all 27 strategies.
// coeffs: `size` floats in the reference coefficient layout (clobbered copy);
// pixels: rows x cols floats with the given stride.
// ---------------------------------------------------------------------------
REF_API int ref_transform_to_pixels(int strategy, const float* coeffs, size_t ncoeff,
                                    float* pixels, size_t stride) {
  JxlMemoryManager mm;
  if (!MemoryManagerInit(&mm, nullptr)) return 1;
  auto mem = AlignedMemory::Create(&mm, (ncoeff + 5 * AcStrategy::kMaxCoeffArea) * sizeof(float));
  if (!mem.ok()) return 2;
  AlignedMemory m = std::move(mem).value_();
  float* c = m.address<float>();
  float* scratch = c + ncoeff;
  memcpy(c, coeffs, ncoeff * sizeof(float));
  TransformToPixels(static_cast<AcStrategyType>(strategy), c, pixels, stride, scratch);
  return 0;
}

REF_API int ref_transform_from_pixels(int strategy, const float* pixels, size_t stride,
                                      float* coeffs, size_t ncoeff) {
  JxlMemoryManager mm;
  if (!MemoryManagerInit(&mm, nullptr)) return 1;
  auto mem = AlignedMemory::Create(&mm, (ncoeff + 5 * AcStrategy::kMaxCoeffArea) * sizeof(float));
  if (!mem.ok()) return 2;
  AlignedMemory m = std::move(mem).value_();
  float* c = m.address<float>();
  float* scratch = c + ncoeff;
  TransformFromPixels(static_cast<AcStrategyType>(strategy), pixels, stride, c, scratch);
  memcpy(coeffs, c, ncoeff * sizeof(float));
  return 0;
}

// dc: cov_y x cov_x window (stride dc_stride); llf: top-left of a coefficient
// block of the strategy (written with row stride max(cov)*8 by the reference).
REF_API int ref_llf_from_dc(int strategy, const float* dc, size_t dc_stride, float* block,
                            size_t ncoeff) {
  JxlMemoryManager mm;
  if (!MemoryManagerInit(&mm, nullptr)) return 1;
  auto mem = AlignedMemory::Create(&mm, (ncoeff + 5 * AcStrategy::kMaxCoeffArea) * sizeof(float));
  if (!mem.ok()) return 2;
  AlignedMemory m = std::move(mem).value_();
  float* c = m.address<float>();
  float* scratch = c + ncoeff;
  memcpy(c, block, ncoeff * sizeof(float));
  LowestFrequenciesFromDC(static_cast<AcStrategyType>(strategy), dc, dc_stride, c, scratch);
  memcpy(block, c, ncoeff * sizeof(float));
  return 0;
}

// ---------------------------------------------------------------------------
// (6) DC stage, the step right before the hot path (SURVEY.md §8f rank 2):
// DequantDC (lib/jxl/compressed_dc.cc:199-300, 4:4:4 branch) on one DC group and
// AdaptiveDCSmoothing (:128-197) on the whole DC image, with the reference's code.
// q[c]: quantised DC planes xs*ys in X, Y, B order; out/dc: [3][ys][xs] floats.
// ---------------------------------------------------------------------------
REF_API int ref_dequant_dc(const int32_t* const q[3], size_t xs, size_t ys, const float* dc_factors, float mul,
                           const float* cfl_factors, float* out) {
  JxlMemoryManager mm;
  if (!MemoryManagerInit(&mm, nullptr)) return 1;
  auto img = Image::Create(&mm, xs, ys, 16, 3);
  auto dc = Image3F::Create(&mm, xs, ys);
  auto qdc = ImageB::Create(&mm, xs, ys);
  if (!img.ok() || !dc.ok() || !qdc.ok()) return 2;
  Image image = std::move(img).value_();
  Image3F dc3 = std::move(dc).value_();
  ImageB quant_dc = std::move(qdc).value_();
  for (size_t c = 0; c < 3; c++) {
    Channel& ch = image.channel[c < 2 ? c ^ 1 : c];  // modular channel order is Y, X, B (dec_modular.cc:448)
    for (size_t y = 0; y < ys; y++) memcpy(ch.plane.Row(y), q[c] + y * xs, xs * sizeof(int32_t));
  }
  BlockCtxMap bctx;
  YCbCrChromaSubsampling cs;
  DequantDC(Rect(0, 0, xs, ys), &dc3, &quant_dc, image, dc_factors, mul, cfl_factors, cs, bctx);
  for (size_t c = 0; c < 3; c++)
    for (size_t y = 0; y < ys; y++) memcpy(out + (c * ys + y) * xs, dc3.ConstPlaneRow(c, y), xs * sizeof(float));
  return 0;
}

REF_API int ref_adaptive_dc_smoothing(const float* dc_factors, float* dc, size_t xs, size_t ys, int threads) {
  JxlMemoryManager mm;
  if (!MemoryManagerInit(&mm, nullptr)) return 1;
  auto im = Image3F::Create(&mm, xs, ys);
  if (!im.ok()) return 2;
  Image3F dc3 = std::move(im).value_();
  for (size_t c = 0; c < 3; c++)
    for (size_t y = 0; y < ys; y++) memcpy(dc3.PlaneRow(c, y), dc + (c * ys + y) * xs, xs * sizeof(float));
  void* runner = threads > 1 ? JxlThreadParallelRunnerCreate(nullptr, threads) : nullptr;
  ThreadPool pool(runner ? JxlThreadParallelRunner : nullptr, runner);
  Status st = AdaptiveDCSmoothing(&mm, dc_factors, &dc3, &pool);
  if (runner) JxlThreadParallelRunnerDestroy(runner);
  if (!st) return 3;
  for (size_t c = 0; c < 3; c++)
    for (size_t y = 0; y < ys; y++) memcpy(dc + (c * ys + y) * xs, dc3.ConstPlaneRow(c, y), xs * sizeof(float));
  return 0;
}

#ifdef JXLB_REF_HARNESS_GPU
// "gpu" variant only (oracle/build_ref.py): how many frames the compiled-in jxl_b200 backend rendered
extern "C" unsigned long long jxlb_gpu_backend_frames_taken(void);
REF_API unsigned long long ref_gpu_frames_taken() { return jxlb_gpu_backend_frames_taken(); }
#endif

REF_API const char* ref_version() { return "libjxl 0.13.0 (reference, oracle/_ref)"; }

// The Highway target HWY_DYNAMIC_DISPATCH selects on this CPU: the best compiled-in target among the
// supported ones (hwy/targets.h: lower bit = better target).  bench.py states it beside the CPU numbers.
REF_API const char* ref_hwy_target() {
  const int64_t usable = hwy::SupportedTargets() & HWY_TARGETS;
  if (!usable) return "none";
  return hwy::TargetName(usable & -usable);
}
