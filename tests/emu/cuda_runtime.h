// tests/emu/cuda_runtime.h -- TEST INFRASTRUCTURE: a minimal SIMT emulation shim.
//
// tests/emu/build_emu.py compiles the PRODUCT's CUDA sources (libjxl_b200/csrc/*.cu, *.cuh) for the host
// against this header instead of the CUDA toolkit's: every CUDA thread of a block becomes an OS thread,
// __syncthreads()/__syncwarp()/__shfl_up_sync() are real barriers / exchanges, blocks run one after the
// other, streams are synchronous (work is enqueued in dependency order, so program order is a valid
// schedule).  tests/test_emulated_cuda.py then runs the kernels + the C-ABI host code against the oracle
// on a machine WITHOUT a GPU.  It is slow (hundreds of threads per block) and only meant for small
// frames.  Nothing in the product links or loads this.
#pragma once
#include <algorithm>
#include <atomic>
#include <barrier>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

#define __host__
#define __device__
#define __global__
#define __constant__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __grid_constant__
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static

using std::max;
using std::min;

// ---- vector types ----
struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct uint3 { unsigned x, y, z; };
inline float2 make_float2(float x, float y) { return {x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return {x, y, z, w}; }
inline uint2 make_uint2(unsigned x, unsigned y) { return {x, y}; }
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return {x, y, z, w}; }
inline int4 make_int4(int x, int y, int z, int w) { return {x, y, z, w}; }
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};

// ---- per-thread and per-block state ----
inline thread_local uint3 threadIdx, blockIdx;
inline thread_local dim3 blockDim, gridDim;

namespace emu {
struct Warp {
  std::barrier<> bar;
  uint64_t scratch[32];
  unsigned size;
  explicit Warp(int n) : bar(n), size((unsigned)n) {}
};
struct Block {
  std::barrier<> bar;
  std::vector<std::unique_ptr<Warp>> warps;
  void* dyn_smem = nullptr;
  explicit Block(int n) : bar(n) {}
};
inline Block* g_block = nullptr;           // blocks run one at a time
inline thread_local Warp* t_warp = nullptr;
inline thread_local unsigned t_lane = 0;
inline void* dynamic_smem() { return g_block->dyn_smem; }
constexpr int kNumSms = 2;                 // what cudaGetDeviceProperties reports
}  // namespace emu

inline void __syncthreads() { emu::g_block->bar.arrive_and_wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::t_warp->bar.arrive_and_wait(); }
template <typename T>
inline T __shfl_up_sync(unsigned, T v, unsigned delta) {
  static_assert(sizeof(T) <= 8, "");
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  emu::t_warp->scratch[emu::t_lane] = bits;
  emu::t_warp->bar.arrive_and_wait();
  T r = v;
  if (emu::t_lane >= delta) memcpy(&r, &emu::t_warp->scratch[emu::t_lane - delta], sizeof(T));
  emu::t_warp->bar.arrive_and_wait();
  return r;
}
template <typename T>
inline T __shfl_sync(unsigned, T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "");
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  emu::t_warp->scratch[emu::t_lane] = bits;
  emu::t_warp->bar.arrive_and_wait();
  T r;
  memcpy(&r, &emu::t_warp->scratch[src_lane & 31], sizeof(T));
  emu::t_warp->bar.arrive_and_wait();
  return r;
}
inline unsigned __ballot_sync(unsigned, bool pred) {
  emu::t_warp->scratch[emu::t_lane] = pred ? 1 : 0;
  emu::t_warp->bar.arrive_and_wait();
  unsigned m = 0;
  for (unsigned i = 0; i < emu::t_warp->size; i++) m |= (unsigned)emu::t_warp->scratch[i] << i;
  emu::t_warp->bar.arrive_and_wait();
  return m;
}
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
// A load whose address breaks alignof(T) is a misaligned-address fault on the GPU; x86 does not care, so
// __ldg counts them (emu_misaligned_loads) and copies bytewise instead of faulting.
namespace emu {
inline std::atomic<uint64_t> g_misaligned_loads{0};
}
template <typename T>
inline T __ldg(const T* p) {
  if ((uintptr_t)p % alignof(T)) emu::g_misaligned_loads.fetch_add(1, std::memory_order_relaxed);
  T v;
  memcpy(&v, p, sizeof(T));
  return v;
}
// the number of misaligned __ldg loads since the last reset (reset != 0: start counting from zero again)
extern "C" __attribute__((visibility("default"), used)) inline uint64_t emu_misaligned_loads(int reset) {
  return reset ? emu::g_misaligned_loads.exchange(0) : emu::g_misaligned_loads.load();
}
template <typename T>
inline T atomicAdd(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline int __float2int_rn(float x) { return (int)lrintf(x); }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fsqrt_rn(float a) { return sqrtf(a); }
inline float __frcp_rn(float a) { return 1.0f / a; }

// ---- runtime API (synchronous) ----
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2 };
typedef struct emu_stream* cudaStream_t;
typedef struct emu_event* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocDefault = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaDeviceProp { int multiProcessorCount; char name[64]; };
inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
  p->multiProcessorCount = emu::kNumSms;
  snprintf(p->name, sizeof(p->name), "SIMT emulation (host)");
  return cudaSuccess;
}
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
// exact sizes (no rounding up): a sanitizer build then flags even a one-byte overrun of a "device" buffer
inline cudaError_t cudaMalloc(void** p, size_t n) { return posix_memalign(p, 256, n ? n : 1) == 0 ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return posix_memalign(p, 256, n ? n : 1) == 0 ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t = nullptr) {
  for (size_t y = 0; y < h; y++) memcpy((char*)d + y * dp, (const char*)s + y * sp, w);
  return cudaSuccess;
}
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)malloc(1); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (cudaEvent_t)malloc(1); return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = (cudaEvent_t)malloc(1); return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return cudaSuccess; }
template <typename K>
inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int) { return cudaSuccess; }
template <typename K>
inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, K, int, size_t) { *n = 1; return cudaSuccess; }

// ---- kernel launch: KERNEL<<<grid, block, smem, stream>>>(args) is rewritten by build_emu.py into
//      EMU_LAUNCH((KERNEL), grid, block, smem, stream, args) ----
namespace emu {
template <typename K, typename... A>
void launch(K kernel, dim3 grid, dim3 block, size_t smem, A... args) {
  const unsigned nthreads = block.x * block.y * block.z;
  const unsigned nwarps = (nthreads + 31) / 32;
  std::vector<char> dyn(smem + 64);
  for (unsigned bz = 0; bz < grid.z; bz++)
    for (unsigned by = 0; by < grid.y; by++)
      for (unsigned bx = 0; bx < grid.x; bx++) {
        Block blk((int)nthreads);
        blk.dyn_smem = (void*)(((uintptr_t)dyn.data() + 63) & ~(uintptr_t)63);
        for (unsigned w = 0; w < nwarps; w++)
          blk.warps.emplace_back(new Warp((int)std::min(32u, nthreads - 32 * w)));
        g_block = &blk;
        std::vector<std::thread> threads;
        threads.reserve(nthreads);
        for (unsigned t = 0; t < nthreads; t++)
          threads.emplace_back([&, t] {
            threadIdx = {t % block.x, (t / block.x) % block.y, t / (block.x * block.y)};
            blockIdx = {bx, by, bz};
            blockDim = block;
            gridDim = grid;
            t_warp = blk.warps[t / 32].get();
            t_lane = t % 32;
            kernel(args...);
            // an exited thread no longer takes part in barriers (as on the GPU)
            t_warp->bar.arrive_and_drop();
            blk.bar.arrive_and_drop();
          });
        for (auto& th : threads) th.join();
        g_block = nullptr;
      }
}
}  // namespace emu
#define EMU_LAUNCH(kernel, grid, block, smem, stream, ...) \
  emu::launch(kernel, dim3(grid), dim3(block), (size_t)(smem), ##__VA_ARGS__)
