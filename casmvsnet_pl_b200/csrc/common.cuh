// Shared helpers for libcasmvs (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
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

// Layout bits of the tensor-core conv launchers (ConvArgs::layout): the input, or the
// output and the skip, stored blocked by channel quads (B, C/4, D, H, W, 4) instead of
// channels-last (B, D, H, W, C).  Only the CostRegNet driver passes them; see DESIGN.md §2.
constexpr int kLayoutXBlocked = 1, kLayoutYBlocked = 2;

// A convolution layer (input dims) for a tensor-core launcher, which returns 0 or <0 (error).
// The coverage tables of conv3d_tma.cu and conv3d_tma2.cu map layer shapes to launchers.
struct ConvArgs {
  const float *x, *wpk, *scale, *shift, *skip;
  float* y;
  float slope;
  int B, Cin, Cout, D, h, w, layout, round_out;
};
using ConvLauncher = int (*)(const ConvArgs& a, cudaStream_t st);

// CostRegNet's conv11 + prob as one kernel (conv3d_tail.cu), blocked activations only.
struct TailArgs {
  const float *u9, *c0;                  // (B,4,D/2,h/2,w/2,4), (B,2,D,h,w,4)
  const float *w11, *scale11, *shift11;  // conv11: packed weights, folded norm
  const float *wp, *scalep, *shiftp;     // prob: packed weights, scale (1) and bias
  float* logits;                         // (B,D,h,w)
  float slope;                           // conv11's LeakyReLU slope
  int B, D, h, w;                        // full resolution, multiples of 8
};
using TailLauncher = int (*)(const TailArgs& a, cudaStream_t st);

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

// Entry-point check of a device pointer that the kernels behind it access in `bytes`-wide
// vectors (null passes: the null checks come after).
#define CASMVS_REQUIRE_ALIGNED(what, ptr, bytes)                                              \
  CASMVS_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & ((bytes) - 1)) == 0,                     \
                 "%s: %s must be %d-byte aligned (got %p)", what, #ptr, (int)(bytes),         \
                 (const void*)(ptr))

// The environment switches of DESIGN.md §5, read once per process: the function-local static
// is initialised on first use, thread-safely.
struct Switches { bool k1_smem, k3_reg, pdl; int tma_dchunk; };
inline const Switches& switches() {
  static const Switches s = [] {
    auto get = [](const char* name, int unset) {
      const char* e = getenv(name);
      return e ? atoi(e) : unset;
    };
    return Switches{get("CASMVS_K1_SMEM", 1) != 0, get("CASMVS_K3_REG", 1) != 0,
                    get("CASMVS_PDL", 1) != 0, get("CASMVS_TMA_DCHUNK", 0)};
  }();
  return s;
}

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
