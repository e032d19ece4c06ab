// K3 — softmax over the D hypotheses + soft-argmax depth + index + confidence,
// K4 — depth hypotheses for the next cascade stage.
//
// Inverse-depth plane sweep (opt-in; README "Wide depth ranges").  Stage l in {2,1,0} (2 the
// coarsest) has D_l planes and interval ratio r_l; m = init_depth_min, i = depth_interval.
//   1. near n = m, far f = m + (D_2-1)*i*r_2 in float32 as uniform_hypotheses_kernel forms its
//      last plane; n > 0, f > n, both finite, or the call is refused (ops.inverse_steps).
//   2. In double per batch item, each rounded once to float32: u_near = 1/n, u_far = 1/f,
//      s_2 = (1/n - 1/f)/(D_2-1), s_l = s_2*r_l/r_2.
//   3. Coarsest stage: u_k = u_near - s_2*k, d_k = RN(1/u_k) (inverse_plane, k1_common.cuh).
//   4. Finer stages: c = the previous depth upsampled x2 (upsample2x_at), u_c = RN(1/c),
//      u_0 = max(u_c + (D_l/2)*s_l, u_far + (D_l-1)*s_l), u_k = u_0 - s_l*k, d_k = RN(1/u_k).
//      The clamp keeps every plane on this side of the far plane, so every u_k stays positive.
//   5. K3: ubar = sum_k p_k*RN(1/d_k) in the order the uniform kernel sums p_k*d_k, depth =
//      RN(1/ubar); index and confidence unchanged.  Backward (backward.cu):
//      d depth / d logit_k = -depth^2 * p_k * (RN(1/d_k) - ubar) * grad.
// Every product, sum and difference above is one float32 operation rounded to nearest; depth is
// increasing in k as in the uniform mode.
//
// Adaptive depth ranges (opt-in; README "Adaptive depth ranges"; after UCS-Net, Cheng et al.,
// CVPR 2020).  Stage l has D_l planes; g_l = depth_interval*r_l is the uniform mode's step.
//   1. Coarsest stage: the uniform planes, init_depth_min + k*g_2.
//   2. Spread: after stage l+1 (l+1 in {2,1}) regresses dhat = sum_k p_k*d_k, K3 also writes
//      sigma = sqrt_rn(sum_k RN(p_k * RN(RN(d_k - dhat)^2))), a second pass over the planes with
//      the same float32 p_k, summed in the plane order and Cascade16 structure of the depth sum
//      (never E[d^2] - dhat^2, which cancels at DTU depths).  Depth, confidence and index are
//      unchanged.  The finest stage writes no spread.
//   3. Finer stage l in {1,0}: c = upsample2x_at(dhat_{l+1}), s = upsample2x_at(sigma_{l+1}),
//      r = fmaxf(RN(lambda*s), g_l) with lambda = kAdaptiveLambda = 1.5, lo = fmaxf(RN(c - r),
//      1e-7f), hi = RN(c + r), step = RN(RN(hi - lo) / (D_l - 1)) (IEEE division), and plane k
//      is RN(lo + RN(step*k)), the uniform ladder's expression with a per-pixel first and step.
//      The floor keeps a confident pixel searching at least +-g_l; fmaxf ignores NaN, so a NaN
//      spread gives r = g_l, while a NaN c propagates as in the uniform mode.  D_l >= 2.
//   4. Regression, confidence and the backward are the uniform mode's; sigma carries no gradient.
//
// Replaces (reference, relative to /root/reference):
//   F.softmax + depth_regression    models/mvsnet.py:174-177, models/modules.py:95-104
//   confidence block                models/mvsnet.py:179-193
//   get_depth_values                models/modules.py:34-49
//   x2 bilinear upsample            models/mvsnet.py:231-234
//   initial uniform planes          models/mvsnet.py:213-229
#include "k1_common.cuh"

namespace casmvs {

constexpr int kK3Threads = 128;
// lambda of the adaptive mode (rule 3 above), ops.ADAPTIVE_LAMBDA on the Python side
constexpr float kAdaptiveLambda = 1.5f;

// What K3 averages for plane depth x: x itself, or RN(1/x) in the inverse mode.
template <bool INV>
__device__ __forceinline__ float plane_value(float x) {
  if constexpr (INV) return __frcp_rn(x);
  else return x;
}

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
// INV: inverse-depth regression (rule 5 above).  SPREAD: the adaptive mode's spread (rule 2 of
// "Adaptive depth ranges"), written where `spread` is not null; PIX: the per-pixel-step ladder.
// The body of regress_kernel (uniform), regress_inv_kernel and regress_spread_kernel; the uniform
// kernel keeps its name and its code.
template <bool IS_PROB, int DT, bool INV, bool SPREAD = false, bool PIX = false>
__device__ __forceinline__ void
regress_body(const float* __restrict__ logits, const float* __restrict__ dv, int dv_is_vector,
             const Hyp hyp, float* __restrict__ depth, float* __restrict__ conf,
             long long* __restrict__ index, float* __restrict__ prob, int D, int hw,
             float* __restrict__ spread = nullptr) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= hw) return;
  const float* lp = logits + (size_t)b * D * hw + pix;
  // hypotheses: (D,) vector, (B,D,h,w) tensor, or (dv == null) the ladder first + step*d
  const float* dp = !dv ? nullptr : dv_is_vector ? dv : dv + (size_t)b * D * hw + pix;
  const size_t dstride = dv_is_vector ? 1 : (size_t)hw;
  const HypPixT<INV, PIX> hp(hyp, b, D, (size_t)hw, pix);

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
      acc_depth.add(__fmul_rn(p, plane_value<INV>(dp ? __ldg(dp + d * dstride) : hp.at(d))));
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
      acc_depth.add(__fmul_rn(p, plane_value<INV>(dp ? __ldg(dp + d * dstride) : hp.at(d))));
      acc_idx.add(__fmul_rn(p, (float)d));
    }
  }
  const float dep = INV ? __frcp_rn(acc_depth.result()) : acc_depth.result();
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
  if constexpr (SPREAD) {
    // second pass with the same p_k and d_k, now that dep is known
    if (!spread) return;
    Cascade16 acc_var;
    for (int d = 0; d < D; ++d) {
      float p = __ldg(lp + (size_t)d * hw);
      if (!IS_PROB) p = __fdiv_rn(expf(p - m), denom);
      const float t = __fsub_rn(dp ? __ldg(dp + d * dstride) : hp.at(d), dep);
      acc_var.add(__fmul_rn(p, __fmul_rn(t, t)));
    }
    spread[(size_t)b * hw + pix] = __fsqrt_rn(acc_var.result());
  }
}

template <bool IS_PROB, int DT>
__global__ void __launch_bounds__(kK3Threads)
regress_kernel(const float* __restrict__ logits, const float* __restrict__ dv, int dv_is_vector,
               const Hyp hyp, float* __restrict__ depth, float* __restrict__ conf,
               long long* __restrict__ index, float* __restrict__ prob, int D, int hw) {
  regress_body<IS_PROB, DT, false>(logits, dv, dv_is_vector, hyp, depth, conf, index, prob, D, hw);
}
template <bool IS_PROB, int DT>
__global__ void __launch_bounds__(kK3Threads)
regress_inv_kernel(const float* __restrict__ logits, const float* __restrict__ dv, int dv_is_vector,
                   const Hyp hyp, float* __restrict__ depth, float* __restrict__ conf,
                   long long* __restrict__ index, float* __restrict__ prob, int D, int hw) {
  regress_body<IS_PROB, DT, true>(logits, dv, dv_is_vector, hyp, depth, conf, index, prob, D, hw);
}
// regress_kernel with the adaptive mode's spread (null: none) and, PIX, a per-pixel-step ladder
template <bool IS_PROB, int DT, bool PIX>
__global__ void __launch_bounds__(kK3Threads)
regress_spread_kernel(const float* __restrict__ logits, const float* __restrict__ dv,
                      int dv_is_vector, const Hyp hyp, float* __restrict__ depth,
                      float* __restrict__ conf, long long* __restrict__ index,
                      float* __restrict__ prob, float* __restrict__ spread, int D, int hw) {
  regress_body<IS_PROB, DT, false, true, PIX>(logits, dv, dv_is_vector, hyp, depth, conf, index,
                                              prob, D, hw, spread);
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

// The inverse-depth variant of regress_par_kernel (rule 5 above), the same walk with RN(1/d)
// averaged.  regress_par_kernel keeps its own copy: moved into a shared device function, its
// code (not its results) changed with ptxas's register assignment.  SPREAD / PIX: as in
// regress_body; the spread's terms are formed plane-parallel like T1 and walked by warp 0.
template <bool IS_PROB, bool INV, bool SPREAD = false, bool PIX = false>
__device__ __forceinline__ void
regress_par_body(const float* __restrict__ logits, const float* __restrict__ dv, int dv_is_vector,
                 const Hyp hyp, float* __restrict__ depth, float* __restrict__ conf,
                 long long* __restrict__ index, float* __restrict__ prob, int D, int hw,
                 float* __restrict__ spread = nullptr) {
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
  const HypPixT<INV, PIX> hp(hyp, b, D, (size_t)hw, pix);
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
    T1[d * 32 + p] = __fmul_rn(pr, plane_value<INV>(dp ? __ldg(dp + d * dstride) : hp.at(d)));
    T2[d * 32 + p] = __fmul_rn(pr, (float)d);
    if (prob && valid) prob[(size_t)b * D * hw + (size_t)d * hw + pix] = pr;
  }
  __syncthreads();
  if constexpr (SPREAD) {
    // warp 0 finishes depth, index and confidence (every pixel, valid or not, so that the
    // block meets at the barriers below) and leaves the depth in red[]
    if (s == 0) {
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
      const float dep = acc_depth.result();
      red[p] = dep;
      if (valid) {
        depth[(size_t)b * hw + pix] = dep;
        conf[(size_t)b * hw + pix] = c;
        if (index) index[(size_t)b * hw + pix] = (long long)idx;
      }
    }
    if (!spread) return;                 // the same for the whole block
    __syncthreads();
    const float dep = red[p];
    for (int d = s; d < D; d += kK3Lanes) {
      const float t = __fsub_rn(dp ? __ldg(dp + d * dstride) : hp.at(d), dep);
      T1[d * 32 + p] = __fmul_rn(P[d * 32 + p], __fmul_rn(t, t));
    }
    __syncthreads();
    if (s != 0 || !valid) return;
    Cascade16 acc_var;
    for (int d = 0; d < D; ++d) acc_var.add(T1[d * 32 + p]);
    spread[(size_t)b * hw + pix] = __fsqrt_rn(acc_var.result());
    return;
  }
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
  depth[(size_t)b * hw + pix] = INV ? __frcp_rn(acc_depth.result()) : acc_depth.result();
  conf[(size_t)b * hw + pix] = c;
  if (index) index[(size_t)b * hw + pix] = (long long)idx;
}

template <bool IS_PROB>
__global__ void __launch_bounds__(32 * kK3Lanes)
regress_par_inv_kernel(const float* __restrict__ logits, const float* __restrict__ dv,
                       int dv_is_vector, const Hyp hyp, float* __restrict__ depth,
                       float* __restrict__ conf, long long* __restrict__ index,
                       float* __restrict__ prob, int D, int hw) {
  regress_par_body<IS_PROB, true>(logits, dv, dv_is_vector, hyp, depth, conf, index, prob, D, hw);
}
template <bool IS_PROB, bool PIX>
__global__ void __launch_bounds__(32 * kK3Lanes)
regress_par_spread_kernel(const float* __restrict__ logits, const float* __restrict__ dv,
                          int dv_is_vector, const Hyp hyp, float* __restrict__ depth,
                          float* __restrict__ conf, long long* __restrict__ index,
                          float* __restrict__ prob, float* __restrict__ spread, int D, int hw) {
  regress_par_body<IS_PROB, false, true, PIX>(logits, dv, dv_is_vector, hyp, depth, conf, index,
                                              prob, D, hw, spread);
}

// Pixel pix of (h,w) from the (B,h/2,w/2) map cur upsampled x2, bilinear with
// align_corners=True: src = dst*(in-1)/(out-1).
__device__ __forceinline__ float upsample2x_at(const float* __restrict__ cur, int b, int h, int w,
                                               int pix) {
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
  return __fadd_rn(__fmul_rn(1.f - ly, top), __fmul_rn(ly, bot));
}

// out[b,d,y,x] = max(cur - half_range, 1e-7) + step*d, cur optionally upsampled x2.
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
    c = upsample2x_at(cur, b, h, w, pix);
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

// Inverse-depth planes (rules 3 and 4 above).  cur == null: the coarsest stage, u_0 = u_first;
// otherwise u_0 comes from cur (B,h/2,w/2) upsampled x2 and clamped by u_far.  planes == D
// writes the depths d_k (B,D,h,w); planes == 1 writes u_0 (B,h,w) in 1/depth units, the first
// rung of the ladder that the inverse consumers generate themselves (HypPixT<true>).
__global__ void __launch_bounds__(256)
inverse_hypotheses_kernel(const float* __restrict__ cur, float u_first,
                          const float* __restrict__ u_first_dev, float u_far,
                          const float* __restrict__ u_far_dev, float step,
                          const float* __restrict__ step_dev, float* __restrict__ out, int D,
                          int h, int w, int planes) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  if (pix >= hw) return;
  if (step_dev) step = __ldg(step_dev + b);
  float u0;
  if (cur) {
    if (u_far_dev) u_far = __ldg(u_far_dev + b);
    const float uc = __frcp_rn(upsample2x_at(cur, b, h, w, pix));
    u0 = fmaxf(__fadd_rn(uc, __fmul_rn((float)D * 0.5f, step)),
               __fadd_rn(u_far, __fmul_rn((float)(D - 1), step)));
  } else {
    u0 = u_first_dev ? __ldg(u_first_dev + b) : u_first;
  }
  float* op = out + (size_t)b * planes * hw + pix;
  if (planes == 1) {
    *op = u0;
    return;
  }
  for (int d = 0; d < D; ++d) op[(size_t)d * hw] = inverse_plane(u0, step, d);
}

// Adaptive planes (rule 3 of "Adaptive depth ranges" above) from the previous stage's depth cur
// and spread, both (B,h/2,w/2) and upsampled x2.  step / step_dev: g_l, a scalar or (B) device
// values.  planes == D writes the planes (B,D,h,w) to out; planes == 1 writes the ladder's first
// rung lo to out and its step to step_out, both (B,h,w).
__global__ void __launch_bounds__(256)
adaptive_hypotheses_kernel(const float* __restrict__ cur, const float* __restrict__ spread,
                           float step, const float* __restrict__ step_dev, float* __restrict__ out,
                           float* __restrict__ step_out, int D, int h, int w, int planes) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  if (pix >= hw) return;
  if (step_dev) step = __ldg(step_dev + b);
  const float c = upsample2x_at(cur, b, h, w, pix);
  const float r = fmaxf(__fmul_rn(kAdaptiveLambda, upsample2x_at(spread, b, h, w, pix)), step);
  const float lo = fmaxf(__fsub_rn(c, r), 1e-7f);
  const float hi = __fadd_rn(c, r);
  const float st = __fdiv_rn(__fsub_rn(hi, lo), (float)(D - 1));
  if (planes == 1) {
    out[(size_t)b * hw + pix] = lo;
    step_out[(size_t)b * hw + pix] = st;
    return;
  }
  float* op = out + (size_t)b * D * hw + pix;
  for (int d = 0; d < D; ++d) op[(size_t)d * hw] = __fadd_rn(lo, __fmul_rn(st, (float)d));
}

}  // namespace casmvs

using namespace casmvs;

template <bool INV>
static int regress_impl(const float* logits, const float* depth_values, int dv_is_vector,
                        const Hyp& hyp, int input_is_prob, float* depth, float* confidence,
                        int64_t* index, float* prob, int B, int D, int h, int w, void* stream) {
  constexpr auto k8p = INV ? regress_inv_kernel<true, 8> : regress_kernel<true, 8>;
  constexpr auto k8l = INV ? regress_inv_kernel<false, 8> : regress_kernel<false, 8>;
  constexpr auto kpp = INV ? regress_par_inv_kernel<true> : regress_par_kernel<true>;
  constexpr auto kpl = INV ? regress_par_inv_kernel<false> : regress_par_kernel<false>;
  constexpr auto k0p = INV ? regress_inv_kernel<true, 0> : regress_kernel<true, 0>;
  constexpr auto k0l = INV ? regress_inv_kernel<false, 0> : regress_kernel<false, 0>;
  CASMVS_REQUIRE(logits && depth && confidence, "regress: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "regress: bad dims");
  if (B == 0) return 0;
  const int hw = h * w;
  cudaStream_t st = as_stream(stream);
  const bool par_path = switches().k3_reg;
  const size_t smem = ((size_t)3 * D * 32 + kK3Lanes * 32) * sizeof(float);
  if (D == 8 && par_path) {
    // 8 hypotheses fit a thread's registers and there are plenty of pixels at the finest level:
    // one thread per pixel (about twice as fast as the plane-parallel kernel at 640x512)
    dim3 grd8((hw + kK3Threads - 1) / kK3Threads, B);
    (input_is_prob ? k8p : k8l)<<<grd8, kK3Threads, 0, st>>>(
        logits, depth_values, dv_is_vector, hyp, depth, confidence, (long long*)index, prob, D, hw);
    return after_launch("regress");
  }
  if (par_path && smem <= 96 * 1024) {
    dim3 grd((hw + 31) / 32, B);
    if (input_is_prob) {
      static std::atomic<bool> a[kMaxDevices];
      if (int rc = opt_in_smem(kpp, 96 * 1024, a, "regress")) return rc;
      kpp<<<grd, 32 * kK3Lanes, smem, st>>>(
          logits, depth_values, dv_is_vector, hyp, depth, confidence, (long long*)index, prob, D, hw);
    } else {
      static std::atomic<bool> a[kMaxDevices];
      if (int rc = opt_in_smem(kpl, 96 * 1024, a, "regress")) return rc;
      kpl<<<grd, 32 * kK3Lanes, smem, st>>>(
          logits, depth_values, dv_is_vector, hyp, depth, confidence, (long long*)index, prob, D, hw);
    }
    return after_launch("regress");
  }
  // small maps: narrower blocks so that every SM gets work
  const int threads = (long)hw * B < (long)num_sms() * 4 * kK3Threads ? 32 : kK3Threads;
  dim3 grd((hw + threads - 1) / threads, B);
  (input_is_prob ? k0p : k0l)<<<grd, threads, 0, st>>>(
      logits, depth_values, dv_is_vector, hyp, depth, confidence, (long long*)index, prob, D, hw);
  return after_launch("regress");
}

// The K3 forms of the adaptive mode: the uniform regression plus the spread (null: none) and,
// PIX, the per-pixel-step ladder.  The same path choice as regress_impl.
template <bool PIX>
static int regress_spread_impl(const float* logits, const float* depth_values, int dv_is_vector,
                               const Hyp& hyp, int input_is_prob, float* depth, float* confidence,
                               int64_t* index, float* prob, float* spread, int B, int D, int h,
                               int w, void* stream) {
  CASMVS_REQUIRE(logits && depth && confidence, "regress: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "regress: bad dims");
  if (B == 0) return 0;
  const int hw = h * w;
  cudaStream_t st = as_stream(stream);
  const bool par_path = switches().k3_reg;
  const size_t smem = ((size_t)3 * D * 32 + kK3Lanes * 32) * sizeof(float);
  // a ladder is never a probability input: the per-pixel-step kernels exist for logits only
  auto pick = [input_is_prob](auto kp, auto kl) { return input_is_prob ? kp : kl; };
  if (D == 8 && par_path) {
    const auto k = PIX ? regress_spread_kernel<false, 8, true>
                       : pick(regress_spread_kernel<true, 8, false>, regress_spread_kernel<false, 8, false>);
    dim3 grd8((hw + kK3Threads - 1) / kK3Threads, B);
    k<<<grd8, kK3Threads, 0, st>>>(logits, depth_values, dv_is_vector, hyp, depth, confidence,
                                   (long long*)index, prob, spread, D, hw);
    return after_launch("regress");
  }
  if (par_path && smem <= 96 * 1024) {
    const auto k = PIX ? regress_par_spread_kernel<false, true>
                       : pick(regress_par_spread_kernel<true, false>, regress_par_spread_kernel<false, false>);
    static std::atomic<bool> a[3][kMaxDevices];
    if (int rc = opt_in_smem(k, 96 * 1024, a[PIX ? 2 : input_is_prob ? 1 : 0], "regress")) return rc;
    dim3 grd((hw + 31) / 32, B);
    k<<<grd, 32 * kK3Lanes, smem, st>>>(logits, depth_values, dv_is_vector, hyp, depth, confidence,
                                        (long long*)index, prob, spread, D, hw);
    return after_launch("regress");
  }
  const auto k = PIX ? regress_spread_kernel<false, 0, true>
                     : pick(regress_spread_kernel<true, 0, false>, regress_spread_kernel<false, 0, false>);
  const int threads = (long)hw * B < (long)num_sms() * 4 * kK3Threads ? 32 : kK3Threads;
  dim3 grd((hw + threads - 1) / threads, B);
  k<<<grd, threads, 0, st>>>(logits, depth_values, dv_is_vector, hyp, depth, confidence,
                             (long long*)index, prob, spread, D, hw);
  return after_launch("regress");
}

extern "C" int casmvs_regress_fwd(const float* logits, const float* depth_values,
                                  int dv_is_vector, int input_is_prob, float* depth,
                                  float* confidence, int64_t* index, float* prob, int B, int D,
                                  int h, int w, void* stream) {
  CASMVS_REQUIRE(depth_values, "regress: null pointer");
  CASMVS_REQUIRE((input_is_prob & ~(1 | CASMVS_INVERSE_DEPTH)) == 0, "regress: bad input_is_prob flags");
  const Hyp hyp{depth_values, nullptr, nullptr, nullptr, 0.f, 0.f};
  const int is_prob = input_is_prob & 1;
  if (input_is_prob & CASMVS_INVERSE_DEPTH)
    return regress_impl<true>(logits, depth_values, dv_is_vector, hyp, is_prob, depth, confidence,
                              index, prob, B, D, h, w, stream);
  return regress_impl<false>(logits, depth_values, dv_is_vector, hyp, is_prob, depth, confidence,
                             index, prob, B, D, h, w, stream);
}

// Cascade-internal variant: hypotheses = first + step*d (Hyp, k1_common.cuh), never materialised.
extern "C" int casmvs_regress_ladder_fwd(const float* logits, const float* first_map,
                                         const float* first_b, float first, const float* step_b,
                                         float step, float* depth, float* confidence,
                                         int64_t* index, int B, int D, int h, int w, void* stream) {
  const Hyp hyp{nullptr, first_map, first_b, step_b, first, step};
  return regress_impl<false>(logits, nullptr, 0, hyp, 0, depth, confidence, index, nullptr, B, D, h,
                             w, stream);
}

// The same over the inverse-depth ladder: hypotheses 1/(first - step*d), inverse regression.
extern "C" int casmvs_regress_ladder_inverse_fwd(const float* logits, const float* first_map,
                                                 const float* first_b, float first,
                                                 const float* step_b, float step, float* depth,
                                                 float* confidence, int64_t* index, int B, int D,
                                                 int h, int w, void* stream) {
  const Hyp hyp{nullptr, first_map, first_b, step_b, first, step};
  return regress_impl<true>(logits, nullptr, 0, hyp, 0, depth, confidence, index, nullptr, B, D, h,
                            w, stream);
}

// casmvs_regress_fwd (uniform regression only) that also writes the spread (B,h,w).
extern "C" int casmvs_regress_spread_fwd(const float* logits, const float* depth_values,
                                         int dv_is_vector, int input_is_prob, float* depth,
                                         float* confidence, int64_t* index, float* prob,
                                         float* spread, int B, int D, int h, int w, void* stream) {
  CASMVS_REQUIRE(depth_values && spread, "regress_spread: null pointer");
  CASMVS_REQUIRE((input_is_prob & ~1) == 0, "regress_spread: bad input_is_prob flags");
  const Hyp hyp{depth_values, nullptr, nullptr, nullptr, 0.f, 0.f};
  return regress_spread_impl<false>(logits, depth_values, dv_is_vector, hyp, input_is_prob, depth,
                                    confidence, index, prob, spread, B, D, h, w, stream);
}

// casmvs_regress_ladder_fwd with the spread (may be null only with step_map) and the per-pixel
// step: step_map (B,h,w) non-null takes the ladder first_map + step_map*d (first_map required).
extern "C" int casmvs_regress_ladder_spread_fwd(const float* logits, const float* first_map,
                                                const float* first_b, float first,
                                                const float* step_b, float step,
                                                const float* step_map, float* depth,
                                                float* confidence, int64_t* index, float* spread,
                                                int B, int D, int h, int w, void* stream) {
  if (step_map) {
    CASMVS_REQUIRE(first_map, "regress_ladder_spread: a step map needs a first map");
    const Hyp hyp{nullptr, first_map, nullptr, step_map, 0.f, 0.f};
    return regress_spread_impl<true>(logits, nullptr, 0, hyp, 0, depth, confidence, index, nullptr,
                                     spread, B, D, h, w, stream);
  }
  CASMVS_REQUIRE(spread, "regress_ladder_spread: null spread without a step map");
  const Hyp hyp{nullptr, first_map, first_b, step_b, first, step};
  return regress_spread_impl<false>(logits, nullptr, 0, hyp, 0, depth, confidence, index, nullptr,
                                    spread, B, D, h, w, stream);
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

extern "C" int casmvs_inverse_hypotheses_fwd(const float* cur, float u_first, const float* u_first_dev,
                                             float u_far, const float* u_far_dev, float step,
                                             const float* step_dev, float* out, int planes, int B,
                                             int D, int h, int w, void* stream) {
  CASMVS_REQUIRE(out, "inverse_hypotheses: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "inverse_hypotheses: bad dims");
  CASMVS_REQUIRE(planes == D || (planes == 1 && cur), "inverse_hypotheses: planes must be D, or 1 "
                 "with cur");
  CASMVS_REQUIRE(!cur || (h % 2 == 0 && w % 2 == 0), "inverse_hypotheses: upsample needs even h,w");
  if (B == 0) return 0;
  dim3 grd((h * w + 255) / 256, B);
  inverse_hypotheses_kernel<<<grd, 256, 0, as_stream(stream)>>>(
      cur, u_first, u_first_dev, u_far, u_far_dev, step, step_dev, out, D, h, w, planes);
  return after_launch("inverse_hypotheses");
}

extern "C" int casmvs_adaptive_hypotheses_fwd(const float* cur, const float* spread, float step,
                                              const float* step_dev, float* out, float* step_out,
                                              int planes, int B, int D, int h, int w,
                                              void* stream) {
  CASMVS_REQUIRE(cur && spread && out, "adaptive_hypotheses: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D >= 2 && h > 0 && w > 0,
                 "adaptive_hypotheses: bad dims (D >= 2)");
  CASMVS_REQUIRE(planes == D || (planes == 1 && step_out),
                 "adaptive_hypotheses: planes must be D, or 1 with step_out");
  CASMVS_REQUIRE(h % 2 == 0 && w % 2 == 0, "adaptive_hypotheses: upsample needs even h,w");
  if (B == 0) return 0;
  dim3 grd((h * w + 255) / 256, B);
  adaptive_hypotheses_kernel<<<grd, 256, 0, as_stream(stream)>>>(cur, spread, step, step_dev, out,
                                                                 step_out, D, h, w, planes);
  return after_launch("adaptive_hypotheses");
}
