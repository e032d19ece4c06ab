// K3 — softmax over the D hypotheses + soft-argmax depth + index + confidence,
// K4 — depth hypotheses for the next cascade stage.
//
// Replaces (reference, relative to /root/reference):
//   F.softmax + depth_regression    models/mvsnet.py:174-177, models/modules.py:95-104
//   confidence block                models/mvsnet.py:179-193
//   get_depth_values                models/modules.py:34-49
//   x2 bilinear upsample            models/mvsnet.py:231-234
//   initial uniform planes          models/mvsnet.py:213-229
#include <stdlib.h>

#include "k1_common.cuh"

namespace casmvs {

constexpr int kK3Threads = 128;

// Accumulator following the main path of torch-CPU's sum over a non-innermost dim
// for sizes < 256 (ATen SumKernel multi_row_sum, level_step 16): 16 terms are added
// sequentially into acc0, which is then folded into acc1 and cleared; the tail
// stays in acc0; result = acc0 + acc1.  (ATen's tail-vector columns use a 4-way
// interleaved variant, so torch itself is not order-uniform across pixels.)
// __fadd_rn keeps ptxas from fusing.
struct Cascade16 {
  float a0 = 0.f, a1 = 0.f;
  int n = 0;
  __device__ __forceinline__ void add(float t) {
    a0 = __fadd_rn(a0, t);
    if (++n == 16) { a1 = __fadd_rn(a1, a0); a0 = 0.f; n = 0; }
  }
  __device__ __forceinline__ float result() const { return __fadd_rn(a0, a1); }
};

// DT > 0: D is the compile-time constant DT (the cascade's 8 / 48): the D logits of a
// pixel are loaded ONCE into registers (D independent loads in flight instead of three
// dependent passes over global memory) and exp(l - m) is evaluated once per hypothesis.  The
// arithmetic -- every operation and its order -- is the generic path's, so results are
// bit-identical (tests/test_gpu_kernels.py::test_regress_register_path_bit_identical).
template <bool IS_PROB, int DT>
__global__ void __launch_bounds__(kK3Threads)
regress_kernel(const float* __restrict__ logits, const float* __restrict__ dv, int dv_is_vector,
               const Hyp hyp, float* __restrict__ depth, float* __restrict__ conf,
               long long* __restrict__ index, float* __restrict__ prob, int D, int hw) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= hw) return;
  const float* lp = logits + (size_t)b * D * hw + pix;
  // hypotheses: (D,) vector, (B,D,h,w) tensor, or (dv == null) the ladder first + step*d
  const float* dp = !dv ? nullptr : dv_is_vector ? dv : dv + (size_t)b * D * hw + pix;
  const size_t dstride = dv_is_vector ? 1 : (size_t)hw;
  const HypPix hp(hyp, b, D, (size_t)hw, pix);

  float m = 0.f, denom = 1.f;
  Cascade16 acc_depth, acc_idx;
  if constexpr (DT > 0) {
    float l[DT];
#pragma unroll
    for (int d = 0; d < DT; ++d) l[d] = __ldg(lp + (size_t)d * hw);
    if (!IS_PROB) {
      m = -INFINITY;
#pragma unroll
      for (int d = 0; d < DT; ++d) m = fmaxf(m, l[d]);
      denom = 0.f;
#pragma unroll
      for (int d = 0; d < DT; ++d) {
        l[d] = expf(l[d] - m);
        denom = __fadd_rn(denom, l[d]);
      }
    }
#pragma unroll
    for (int d = 0; d < DT; ++d) {
      float p = l[d];
      if (!IS_PROB) p = __fdiv_rn(p, denom);
      if (prob) prob[(size_t)b * D * hw + (size_t)d * hw + pix] = p;
      acc_depth.add(__fmul_rn(p, dp ? __ldg(dp + d * dstride) : hp.at(d)));
      acc_idx.add(__fmul_rn(p, (float)d));
    }
  } else {
    if (!IS_PROB) {
      m = -INFINITY;
      for (int d = 0; d < D; ++d) m = fmaxf(m, __ldg(lp + (size_t)d * hw));
      denom = 0.f;
      for (int d = 0; d < D; ++d) denom = __fadd_rn(denom, expf(__ldg(lp + (size_t)d * hw) - m));
    }
    for (int d = 0; d < D; ++d) {
      float p = __ldg(lp + (size_t)d * hw);
      if (!IS_PROB) p = __fdiv_rn(expf(p - m), denom);
      if (prob) prob[(size_t)b * D * hw + (size_t)d * hw + pix] = p;
      acc_depth.add(__fmul_rn(p, dp ? __ldg(dp + d * dstride) : hp.at(d)));
      acc_idx.add(__fmul_rn(p, (float)d));
    }
  }
  const float dep = acc_depth.result();
  const float fidx = acc_idx.result();
  // .long() truncates toward zero; clamp to [0, D-1]  (mvsnet.py:189-190)
  int idx;
  if (!(fidx > 0.f)) idx = 0;                       // also catches NaN
  else if (fidx >= (float)(D - 1)) idx = D - 1;
  else idx = (int)fidx;
  // window [idx-1, idx+2], zero padded, summed front to back like avg_pool3d
  float c = 0.f;
#pragma unroll
  for (int k = -1; k <= 2; ++k) {
    int d = idx + k;
    float p = 0.f;
    if (d >= 0 && d < D) {
      p = __ldg(lp + (size_t)d * hw);
      if (!IS_PROB) p = __fdiv_rn(expf(p - m), denom);
    }
    c = __fadd_rn(c, p);
  }
  depth[(size_t)b * hw + pix] = dep;
  conf[(size_t)b * hw + pix] = c;
  if (index) index[(size_t)b * hw + pix] = (long long)idx;
}

// Plane-parallel variant (the default): the generic kernel above runs ~80 instructions per
// hypothesis in ONE thread per pixel (precise expf, IEEE division, 64-bit addressing) -- at
// 160x128 that is 640 warps with a 3 800-instruction dependent chain each, far too few to hide
// the latency.  Here a block owns 32 pixels and NL = 8 warps split the D
// planes: max, exp, the division and the two products are evaluated plane-parallel; only the
// ORDERED sums (sequential denominator, cascade-16 depth / index) are walked by one warp, from
// shared memory.  Every value and every summation order is the generic kernel's, so the two
// are bit-identical (tests/test_gpu_kernels.py::test_regress_register_path_bit_identical).
constexpr int kK3Lanes = 8;
template <bool IS_PROB>
__global__ void __launch_bounds__(32 * kK3Lanes)
regress_par_kernel(const float* __restrict__ logits, const float* __restrict__ dv, int dv_is_vector,
                   const Hyp hyp, float* __restrict__ depth, float* __restrict__ conf,
                   long long* __restrict__ index, float* __restrict__ prob, int D, int hw) {
  extern __shared__ float sh[];
  float* P = sh;                       // [D][32]  exp, then probability
  float* T1 = sh + (size_t)D * 32;     // [D][32]  p * depth_value
  float* T2 = T1 + (size_t)D * 32;     // [D][32]  p * d
  float* red = T2 + (size_t)D * 32;    // [kK3Lanes][32]
  const int p = threadIdx.x & 31, s = threadIdx.x >> 5;
  const int b = blockIdx.y;
  const int pixr = blockIdx.x * 32 + p;
  const bool valid = pixr < hw;
  const int pix = valid ? pixr : hw - 1;
  const float* lp = logits + (size_t)b * D * hw + pix;
  // hypotheses: (D,) vector, (B,D,h,w) tensor, or (dv == null) the ladder first + step*d
  const float* dp = !dv ? nullptr : dv_is_vector ? dv : dv + (size_t)b * D * hw + pix;
  const size_t dstride = dv_is_vector ? 1 : (size_t)hw;
  const HypPix hp(hyp, b, D, (size_t)hw, pix);
  float m = 0.f;
  if (!IS_PROB) {
    float lmax = -INFINITY;
    for (int d = s; d < D; d += kK3Lanes) {
      const float l = __ldg(lp + (size_t)d * hw);
      P[d * 32 + p] = l;
      lmax = fmaxf(lmax, l);
    }
    red[s * 32 + p] = lmax;
    __syncthreads();
    m = red[p];
#pragma unroll
    for (int k = 1; k < kK3Lanes; ++k) m = fmaxf(m, red[k * 32 + p]);
    for (int d = s; d < D; d += kK3Lanes) P[d * 32 + p] = expf(P[d * 32 + p] - m);
    __syncthreads();
    if (s == 0) {
      float denom = 0.f;
      for (int d = 0; d < D; ++d) denom = __fadd_rn(denom, P[d * 32 + p]);
      red[p] = denom;
    }
    __syncthreads();
  }
  const float denom = IS_PROB ? 1.f : red[p];
  for (int d = s; d < D; d += kK3Lanes) {
    float pr = IS_PROB ? __ldg(lp + (size_t)d * hw) : __fdiv_rn(P[d * 32 + p], denom);
    P[d * 32 + p] = pr;
    T1[d * 32 + p] = __fmul_rn(pr, dp ? __ldg(dp + d * dstride) : hp.at(d));
    T2[d * 32 + p] = __fmul_rn(pr, (float)d);
    if (prob && valid) prob[(size_t)b * D * hw + (size_t)d * hw + pix] = pr;
  }
  __syncthreads();
  if (s != 0 || !valid) return;
  Cascade16 acc_depth, acc_idx;
  for (int d = 0; d < D; ++d) {
    acc_depth.add(T1[d * 32 + p]);
    acc_idx.add(T2[d * 32 + p]);
  }
  const float fidx = acc_idx.result();
  int idx;
  if (!(fidx > 0.f)) idx = 0;
  else if (fidx >= (float)(D - 1)) idx = D - 1;
  else idx = (int)fidx;
  float c = 0.f;
#pragma unroll
  for (int k = -1; k <= 2; ++k) {
    const int d = idx + k;
    c = __fadd_rn(c, (d >= 0 && d < D) ? P[d * 32 + p] : 0.f);
  }
  depth[(size_t)b * hw + pix] = acc_depth.result();
  conf[(size_t)b * hw + pix] = c;
  if (index) index[(size_t)b * hw + pix] = (long long)idx;
}

// out[b,d,y,x] = max(cur - half_range, 1e-7) + step*d, cur optionally upsampled x2
// (align_corners=True: src = dst*(in-1)/(out-1)).
__global__ void __launch_bounds__(256)
hypotheses_kernel(const float* __restrict__ cur, int upsample, float half_range, float step,
                  const float* __restrict__ step_dev, float* __restrict__ out, int D, int h,
                  int w, int planes) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  if (pix >= hw) return;
  float c;
  if (upsample) {
    const int hi = h / 2, wi = w / 2;
    const int y = pix / w, x = pix - y * w;
    const float sy = hi > 1 ? (float)(hi - 1) / (float)(h - 1) : 0.f;
    const float sx = wi > 1 ? (float)(wi - 1) / (float)(w - 1) : 0.f;
    const float fy = sy * (float)y, fx = sx * (float)x;
    int y0 = (int)fy, x0 = (int)fx;
    y0 = min(y0, hi - 1); x0 = min(x0, wi - 1);
    const int y1 = min(y0 + 1, hi - 1), x1 = min(x0 + 1, wi - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const float* cp = cur + (size_t)b * hi * wi;
    const float v00 = __ldg(cp + y0 * wi + x0), v01 = __ldg(cp + y0 * wi + x1);
    const float v10 = __ldg(cp + y1 * wi + x0), v11 = __ldg(cp + y1 * wi + x1);
    const float top = __fadd_rn(__fmul_rn(1.f - lx, v00), __fmul_rn(lx, v01));
    const float bot = __fadd_rn(__fmul_rn(1.f - lx, v10), __fmul_rn(lx, v11));
    c = __fadd_rn(__fmul_rn(1.f - ly, top), __fmul_rn(ly, bot));
  } else {
    c = __ldg(cur + (size_t)b * hw + pix);
  }
  if (step_dev) {
    step = __ldg(step_dev + b);
    half_range = __fmul_rn((float)D * 0.5f, step);
  }
  const float first = fmaxf(__fsub_rn(c, half_range), 1e-7f);
  // planes == D: the full (B,D,h,w) ladder; planes == 1: only its first rung (B,h,w) -- the
  // consumers then generate first + step*d themselves (Hyp, k1_common.cuh)
  float* op = out + (size_t)b * planes * hw + pix;
  for (int d = 0; d < planes; ++d) op[(size_t)d * hw] = __fadd_rn(first, __fmul_rn(step, (float)d));
}

__global__ void __launch_bounds__(256)
uniform_hypotheses_kernel(float depth_min, float step, const float* __restrict__ depth_min_dev,
                          const float* __restrict__ step_dev, float* __restrict__ out, int D,
                          int hw) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= hw) return;
  if (depth_min_dev) depth_min = __ldg(depth_min_dev + b);
  if (step_dev) step = __ldg(step_dev + b);
  float* op = out + (size_t)b * D * hw + pix;
  for (int d = 0; d < D; ++d) op[(size_t)d * hw] = __fadd_rn(depth_min, __fmul_rn(step, (float)d));
}

}  // namespace casmvs

using namespace casmvs;

static int regress_impl(const float* logits, const float* depth_values, int dv_is_vector,
                        const Hyp& hyp, int input_is_prob, float* depth, float* confidence,
                        int64_t* index, float* prob, int B, int D, int h, int w, void* stream) {
  CASMVS_REQUIRE(logits && depth && confidence, "regress: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "regress: bad dims");
  if (B == 0) return 0;
  const int hw = h * w;
  cudaStream_t st = as_stream(stream);
  static int par_path = -1;
  if (par_path < 0) {
    const char* e = getenv("CASMVS_K3_REG");      // 0: the one-thread-per-pixel generic kernel
    par_path = e ? atoi(e) : 1;
  }
  const size_t smem = ((size_t)3 * D * 32 + kK3Lanes * 32) * sizeof(float);
  if (D == 8 && par_path) {
    // 8 hypotheses fit a thread's registers and there are plenty of pixels at the finest level:
    // one thread per pixel (about twice as fast as the plane-parallel kernel at 640x512)
    dim3 grd8((hw + kK3Threads - 1) / kK3Threads, B);
    if (input_is_prob)
      regress_kernel<true, 8><<<grd8, kK3Threads, 0, st>>>(logits, depth_values, dv_is_vector, hyp, depth,
                                                           confidence, (long long*)index, prob, D, hw);
    else
      regress_kernel<false, 8><<<grd8, kK3Threads, 0, st>>>(logits, depth_values, dv_is_vector, hyp, depth,
                                                            confidence, (long long*)index, prob, D, hw);
    return after_launch("regress");
  }
  if (par_path && smem <= 96 * 1024) {
    dim3 grd((hw + 31) / 32, B);
    if (input_is_prob) {
      static std::atomic<bool> a[kMaxDevices];
      if (int rc = opt_in_smem(regress_par_kernel<true>, 96 * 1024, a, "regress")) return rc;
      regress_par_kernel<true><<<grd, 32 * kK3Lanes, smem, st>>>(
          logits, depth_values, dv_is_vector, hyp, depth, confidence, (long long*)index, prob, D, hw);
    } else {
      static std::atomic<bool> a[kMaxDevices];
      if (int rc = opt_in_smem(regress_par_kernel<false>, 96 * 1024, a, "regress")) return rc;
      regress_par_kernel<false><<<grd, 32 * kK3Lanes, smem, st>>>(
          logits, depth_values, dv_is_vector, hyp, depth, confidence, (long long*)index, prob, D, hw);
    }
    return after_launch("regress");
  }
  // small maps: narrower blocks so that every SM gets work
  const int threads = (long)hw * B < (long)num_sms() * 4 * kK3Threads ? 32 : kK3Threads;
  dim3 grd((hw + threads - 1) / threads, B);
  if (input_is_prob)
    regress_kernel<true, 0><<<grd, threads, 0, st>>>(logits, depth_values, dv_is_vector, hyp, depth,
                                                     confidence, (long long*)index, prob, D, hw);
  else
    regress_kernel<false, 0><<<grd, threads, 0, st>>>(logits, depth_values, dv_is_vector, hyp, depth,
                                                      confidence, (long long*)index, prob, D, hw);
  return after_launch("regress");
}

extern "C" int casmvs_regress_fwd(const float* logits, const float* depth_values,
                                  int dv_is_vector, int input_is_prob, float* depth,
                                  float* confidence, int64_t* index, float* prob, int B, int D,
                                  int h, int w, void* stream) {
  CASMVS_REQUIRE(depth_values, "regress: null pointer");
  const Hyp hyp{depth_values, nullptr, nullptr, nullptr, 0.f, 0.f};
  return regress_impl(logits, depth_values, dv_is_vector, hyp, input_is_prob, depth, confidence,
                      index, prob, B, D, h, w, stream);
}

// Cascade-internal variant: hypotheses = first + step*d (Hyp, k1_common.cuh), never materialised.
extern "C" int casmvs_regress_ladder_fwd(const float* logits, const float* first_map,
                                         const float* first_b, float first, const float* step_b,
                                         float step, float* depth, float* confidence,
                                         int64_t* index, int B, int D, int h, int w, void* stream) {
  const Hyp hyp{nullptr, first_map, first_b, step_b, first, step};
  return regress_impl(logits, nullptr, 0, hyp, 0, depth, confidence, index, nullptr, B, D, h, w,
                      stream);
}

extern "C" int casmvs_depth_hypotheses_fwd(const float* cur, int upsample, float half_range,
                                           float step, const float* step_dev, float* out, int B,
                                           int D, int h, int w, void* stream) {
  CASMVS_REQUIRE(cur && out, "depth_hypotheses: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "depth_hypotheses: bad dims");
  CASMVS_REQUIRE(!upsample || (h % 2 == 0 && w % 2 == 0),
                 "depth_hypotheses: upsample needs even h,w");
  if (B == 0) return 0;
  dim3 grd((h * w + 255) / 256, B);
  hypotheses_kernel<<<grd, 256, 0, as_stream(stream)>>>(cur, upsample, half_range, step, step_dev,
                                                        out, D, h, w, D);
  return after_launch("depth_hypotheses");
}

// First rung only: out (B,h,w) = max(cur - half_range, 1e-7), cur optionally upsampled x2.
extern "C" int casmvs_depth_first_fwd(const float* cur, int upsample, float half_range, float step,
                                      const float* step_dev, float* out, int B, int D, int h, int w,
                                      void* stream) {
  CASMVS_REQUIRE(cur && out, "depth_first: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "depth_first: bad dims");
  CASMVS_REQUIRE(!upsample || (h % 2 == 0 && w % 2 == 0), "depth_first: upsample needs even h,w");
  if (B == 0) return 0;
  dim3 grd((h * w + 255) / 256, B);
  hypotheses_kernel<<<grd, 256, 0, as_stream(stream)>>>(cur, upsample, half_range, step, step_dev,
                                                        out, D, h, w, 1);
  return after_launch("depth_first");
}

extern "C" int casmvs_uniform_hypotheses_fwd(float depth_min, float step,
                                             const float* depth_min_dev, const float* step_dev,
                                             float* out, int B, int D, int h, int w,
                                             void* stream) {
  CASMVS_REQUIRE(out, "uniform_hypotheses: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "uniform_hypotheses: bad dims");
  if (B == 0) return 0;
  dim3 grd((h * w + 255) / 256, B);
  uniform_hypotheses_kernel<<<grd, 256, 0, as_stream(stream)>>>(depth_min, step, depth_min_dev,
                                                                step_dev, out, D, h * w);
  return after_launch("uniform_hypotheses");
}
