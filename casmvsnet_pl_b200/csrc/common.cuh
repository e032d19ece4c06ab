// Shared helpers for libcasmvs (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "casmvs.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libcasmvs is written for sm_90a (H100) only"
#endif

namespace casmvs {

// thread-local error string + process-wide launch counter (api.cu)
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
// tensor-core-mode layers that ended on the CUDA-core kernel (casmvs_fallback_count)
extern std::atomic<uint64_t> g_fallbacks;

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Layout bits of the internal conv entry points (conv3d_tma / conv3d_tma2): the input, or the
// output and the skip, stored blocked by channel quads (B, C/4, D, H, W, 4) instead of
// channels-last (B, D, H, W, C).  Only the CostRegNet driver passes them; see DESIGN.md §2.
constexpr int kLayoutXBlocked = 1, kLayoutYBlocked = 2;

// call after every kernel launch: counts it and converts launch errors
inline int after_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: kernel launch failed: %s", what, cudaGetErrorString(e));
    return -2;
  }
  return 0;
}

#define CASMVS_REQUIRE(cond, ...)        \
  do {                                   \
    if (!(cond)) {                       \
      casmvs::set_error(__VA_ARGS__);    \
      return -1;                         \
    }                                    \
  } while (0)

// Host-side state is kept per device ordinal: cudaFuncSetAttribute and the SM count are
// per-device properties, and a process may drive several GPUs (model.to("cuda:1")).
constexpr int kMaxDevices = 64;
inline int cur_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev >= 0 && dev < kMaxDevices ? dev : 0;
}
inline int num_sms() {
  static std::atomic<int> n[kMaxDevices];
  const int dev = cur_device();
  int v = n[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (v <= 0) v = 132;
    n[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}
// cudaFuncAttributeMaxDynamicSharedMemorySize opt-in, once per (kernel, device)
template <typename K>
inline int opt_in_smem(K kfn, int bytes, std::atomic<bool> (&done)[kMaxDevices], const char* what) {
  const int dev = cur_device();
  if (done[dev].load(std::memory_order_acquire)) return 0;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    set_error("%s: cannot opt in to %d B of shared memory: %s", what, bytes, cudaGetErrorString(e));
    return -2;
  }
  done[dev].store(true, std::memory_order_release);
  return 0;
}

// Division of a work-item index by a launch constant without the ~30-instruction runtime
// division: q = umulhi(n, m), m = floor(2^32 / d) + 1, exact while n * d < 2^32 (the host
// checks that with fastdiv_ok before it launches).
struct FastDiv {
  uint32_t d, m;
};
inline FastDiv make_fastdiv(uint32_t d) {
  return FastDiv{d, d > 1 ? (uint32_t)((1ull << 32) / d) + 1u : 0u};
}
inline bool fastdiv_ok(uint64_t n_max, uint32_t d) { return n_max * d < (1ull << 32); }
// n -> n / d, with the remainder in r
__device__ __forceinline__ uint32_t fastdivmod(uint32_t n, const FastDiv f, uint32_t& r) {
  const uint32_t q = f.d > 1 ? __umulhi(n, f.m) : n;
  r = n - q * f.d;
  return q;
}

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}
__device__ __forceinline__ void st4(float* p, float4 v) {
  *reinterpret_cast<float4*>(p) = v;
}
// streaming store: written once, consumed by a later kernel through L2
__device__ __forceinline__ void st4_stream(float* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

}  // namespace casmvs
