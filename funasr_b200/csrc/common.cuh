// Shared helpers for the funasr_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include "../../include/funasr_b200.h"

namespace fa {

extern std::atomic<unsigned long long> g_launch_count;

inline void count_launch(unsigned n = 1) { g_launch_count.fetch_add(n, std::memory_order_relaxed); }

// Returns FA_ERR_CUDA from the enclosing function when the launch that just happened failed.
#define FA_CHECK_LAUNCH()                                        \
  do {                                                           \
    ::fa::count_launch();                                        \
    cudaError_t _e = cudaGetLastError();                         \
    if (_e != cudaSuccess) return FA_ERR_CUDA;                   \
  } while (0)

#define FA_CUDA_OK(expr)                                         \
  do {                                                           \
    cudaError_t _e = (expr);                                     \
    if (_e != cudaSuccess) return FA_ERR_CUDA;                   \
  } while (0)

#define FA_RETURN_IF_ERR(expr)                                   \
  do {                                                           \
    int _s = (expr);                                             \
    if (_s != FA_OK) return _s;                                  \
  } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize and the SM count are PER-DEVICE: a process that drives two GPUs (two handles of
// the offline API, a server with one worker thread per device) must set / query them once per (kernel instantiation, device).
struct PerDeviceOnce { std::atomic<uint32_t> mask{0}; };
template <typename K>
inline int ensure_dyn_smem(K kern, size_t bytes, PerDeviceOnce& once) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return FA_ERR_CUDA;
  const uint32_t bit = 1u << (dev & 31);
  if (!(once.mask.load(std::memory_order_acquire) & bit)) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) return FA_ERR_CUDA;
    once.mask.fetch_or(bit, std::memory_order_release);
  }
  return FA_OK;
}
// SM count of the current device (cached per device)
inline int sm_count() {
  static std::atomic<int> cache[32];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  int n = cache[dev & 31].load(std::memory_order_relaxed);
  if (n <= 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev & 31].store(n, std::memory_order_relaxed);
  }
  return n;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// fp16 planes of a GEMM operand (the x1 / x3 / x6 splits), and of an attention operand (the kernel reads at most two)
static inline int gemm_planes(int mode) { return mode == FA_GEMM_F16X1 ? 1 : (mode == FA_GEMM_F16X3 ? 2 : 3); }
static inline int attn_planes(int mode) { return mode == FA_GEMM_F16X1 ? 1 : 2; }

// Bump allocator over the caller's workspace.  Arena::measuring() runs the same carve without memory: every take succeeds and
// returns a dummy non-null pointer, and bytes() is the workspace size the carve needs — what the *_workspace_bytes queries return.
struct Arena {
  char* base;
  size_t cap, off;
  bool measure = false;
  Arena(void* p, size_t bytes) : base(static_cast<char*>(p)), cap(bytes), off(0) {}
  static Arena measuring() { Arena a(nullptr, SIZE_MAX); a.measure = true; return a; }
  template <typename T>
  T* take(size_t n) {
    size_t o = align_up(off, 256);
    size_t need = n * sizeof(T);
    if (measure) { off = o + need; return reinterpret_cast<T*>(uintptr_t(256)); }
    if (base == nullptr || o + need > cap) { off = cap + 1; return nullptr; }
    off = o + need;
    return reinterpret_cast<T*>(base + o);
  }
  // the next n bytes as an arena of their own: a callee's scratch, which it carves again on every call
  Arena sub(size_t n) { char* p = take<char>(n); return Arena(p, p ? n : 0); }
  bool ok() const { return off <= cap; }
  size_t bytes() const { return off; }
};

}  // namespace fa
