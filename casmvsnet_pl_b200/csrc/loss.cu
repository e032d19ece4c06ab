// Training loss and depth metrics (reference losses.py, metrics.py, train.py:116-122, 145-163).
//
//   loss = sum_l 2^(1-l) * mean over mask_l of smoothL1(pred_l - gt_l)       (beta = 1)
//   metrics (level 0) = sum |e|, #(|e| < 1), #(|e| < 2), #(|e| < 4), n_0
//
// The reference indexes with boolean masks (depth[mask]), which costs a device-to-host sync per
// index on CUDA.  Here the masked reductions are one pass over every level plus one single-block
// pass, with no data-dependent sizes.  Partials are fp64 and reduced in a fixed order (per block,
// then per grid by one block), so the outputs are bit-identical from run to run.
#include "common.cuh"

namespace casmvs {

constexpr int kLossThreads = 256;
constexpr int kLossBlocks = 264;      // fixed: the reduction order must not depend on the device
constexpr int kLossMaxLevels = 4;
// per block: (S_l, n_l) per level, then the four level-0 metric sums
constexpr int kLossSlots = 2 * kLossMaxLevels + 4;

struct LossLevels {
  const float* pred[kLossMaxLevels];
  const float* gt[kLossMaxLevels];
  const uint8_t* mask[kLossMaxLevels];
  float* grad[kLossMaxLevels];
  long long begin[kLossMaxLevels + 1];   // element offsets of each level in the joint index space
  int levels;
};

__device__ __forceinline__ int level_of(const LossLevels& L, long long i) {
  int l = 0;
  while (l + 1 < L.levels && i >= L.begin[l + 1]) ++l;
  return l;
}

// Fixed-order block sum of kLossSlots doubles per thread; result in red[slot * kLossThreads].
__device__ void block_reduce(double (&v)[kLossSlots], double* red) {
  const int t = threadIdx.x;
#pragma unroll
  for (int s = 0; s < kLossSlots; ++s) red[s * kLossThreads + t] = v[s];
  __syncthreads();
  for (int half = kLossThreads / 2; half > 0; half >>= 1) {
    if (t < half) {
#pragma unroll
      for (int s = 0; s < kLossSlots; ++s)
        red[s * kLossThreads + t] += red[s * kLossThreads + t + half];
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kLossThreads) sl1_partials_kernel(LossLevels L, double* partials) {
  __shared__ double red[kLossSlots * kLossThreads];
  double v[kLossSlots];
#pragma unroll
  for (int s = 0; s < kLossSlots; ++s) v[s] = 0.0;
  const long long total = L.begin[L.levels];
  const long long stride = (long long)gridDim.x * kLossThreads;
  for (long long i = (long long)blockIdx.x * kLossThreads + threadIdx.x; i < total; i += stride) {
    const int l = level_of(L, i);
    const long long j = i - L.begin[l];
    if (!L.mask[l][j]) continue;
    const float x = __fsub_rn(L.pred[l][j], L.gt[l][j]);        // depth_pred_l[mask] - gt[mask]
    const double ax = fabs((double)x);
    v[2 * l] += ax < 1.0 ? 0.5 * ax * ax : ax - 0.5;
    v[2 * l + 1] += 1.0;
    if (l == 0) {
      v[2 * kLossMaxLevels + 0] += ax;
      v[2 * kLossMaxLevels + 1] += ax < 1.0 ? 1.0 : 0.0;
      v[2 * kLossMaxLevels + 2] += ax < 2.0 ? 1.0 : 0.0;
      v[2 * kLossMaxLevels + 3] += ax < 4.0 ? 1.0 : 0.0;
    }
  }
  block_reduce(v, red);
  if (threadIdx.x < kLossSlots)
    partials[(size_t)threadIdx.x * kLossBlocks + blockIdx.x] = red[threadIdx.x * kLossThreads];
}

// One block: partials -> loss (fp32), metrics (fp32: sum |e|, acc counts, n_0), counts n_l.
__global__ void __launch_bounds__(kLossThreads) sl1_finish_kernel(const double* partials, int levels,
                                                                  float* loss, float* metrics,
                                                                  long long* counts) {
  __shared__ double red[kLossSlots * kLossThreads];
  double v[kLossSlots];
#pragma unroll
  for (int s = 0; s < kLossSlots; ++s) {
    double acc = 0.0;
    for (int b = threadIdx.x; b < kLossBlocks; b += kLossThreads) acc += partials[(size_t)s * kLossBlocks + b];
    v[s] = acc;
  }
  block_reduce(v, red);
  if (threadIdx.x != 0) return;
  double total = 0.0;
  for (int l = 0; l < levels; ++l) {
    const double n = red[(2 * l + 1) * kLossThreads];
    total += ldexp(1.0, 1 - l) * (red[2 * l * kLossThreads] / n);   // empty mask: 0/0 = NaN
    if (counts) counts[l] = (long long)n;
  }
  if (loss) *loss = (float)total;
  if (metrics) {
    for (int k = 0; k < 4; ++k) metrics[k] = (float)red[(2 * kLossMaxLevels + k) * kLossThreads];
    metrics[4] = (float)red[kLossThreads];
  }
}

// ATen's backward of `smooth_l1_loss(p[m], g[m], reduction='mean') * w` under the sum:
// grad_output = g * w (MulBackward), norm = (float)(1.0 / numel), then per element
// smooth_l1_backward: x <= -1: -norm * go; x >= 1: norm * go; else norm * x * go / beta.
// Unmasked pixels get 0 (IndexBackward scatters into zeros).
__global__ void sl1_bwd_kernel(LossLevels L, const long long* counts, const float* grad_loss) {
  const long long total = L.begin[L.levels];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int l = level_of(L, i);
  const long long j = i - L.begin[l];
  float r = 0.f;
  if (L.mask[l][j]) {
    const float go = __fmul_rn(__ldg(grad_loss), (float)ldexp(1.0, 1 - l));
    const float norm = (float)(1.0 / (double)counts[l]);
    const float x = __fsub_rn(L.pred[l][j], L.gt[l][j]);
    if (x <= -1.f)
      r = __fmul_rn(-norm, go);
    else if (x >= 1.f)
      r = __fmul_rn(norm, go);
    else
      r = __fdiv_rn(__fmul_rn(__fmul_rn(norm, x), go), 1.f);
  }
  L.grad[l][j] = r;
}

static int make_levels(LossLevels& L, const float* const* pred, const float* const* gt,
                       const uint8_t* const* mask, float* const* grad, const int* hw, int B,
                       int levels, const char* what) {
  CASMVS_REQUIRE(pred && gt && mask && hw, "%s: null pointer", what);
  CASMVS_REQUIRE(levels >= 1 && levels <= kLossMaxLevels, "%s: levels must be in 1..%d", what,
                 kLossMaxLevels);
  CASMVS_REQUIRE(B >= 1, "%s: bad batch", what);
  L.levels = levels;
  L.begin[0] = 0;
  for (int l = 0; l < levels; ++l) {
    CASMVS_REQUIRE(pred[l] && gt[l] && mask[l] && (!grad || grad[l]), "%s: null pointer (level %d)",
                   what, l);
    CASMVS_REQUIRE(hw[2 * l] > 0 && hw[2 * l + 1] > 0, "%s: bad dims (level %d)", what, l);
    L.pred[l] = pred[l];
    L.gt[l] = gt[l];
    L.mask[l] = mask[l];
    L.grad[l] = grad ? grad[l] : nullptr;
    L.begin[l + 1] = L.begin[l] + (long long)B * hw[2 * l] * hw[2 * l + 1];
  }
  CASMVS_REQUIRE(L.begin[levels] < (1ll << 40), "%s: too many elements", what);
  return 0;
}

}  // namespace casmvs

using namespace casmvs;

extern "C" size_t casmvs_sl1_loss_workspace_bytes(void) {
  return (size_t)kLossSlots * kLossBlocks * sizeof(double);
}

extern "C" int casmvs_sl1_loss_fwd(const float* const* pred, const float* const* gt,
                                   const uint8_t* const* mask, const int* hw, int B, int levels,
                                   float* loss, float* metrics, long long* counts, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  LossLevels L;
  if (int rc = make_levels(L, pred, gt, mask, nullptr, hw, B, levels, "sl1_loss_fwd")) return rc;
  CASMVS_REQUIRE(loss || metrics || counts, "sl1_loss_fwd: no output");
  CASMVS_REQUIRE(workspace && workspace_bytes >= casmvs_sl1_loss_workspace_bytes(),
                 "sl1_loss_fwd: workspace too small (%zu B needed)", casmvs_sl1_loss_workspace_bytes());
  cudaStream_t st = as_stream(stream);
  double* partials = static_cast<double*>(workspace);
  sl1_partials_kernel<<<kLossBlocks, kLossThreads, 0, st>>>(L, partials);
  if (int rc = after_launch("sl1_partials")) return rc;
  sl1_finish_kernel<<<1, kLossThreads, 0, st>>>(partials, levels, loss, metrics, counts);
  return after_launch("sl1_finish");
}

extern "C" int casmvs_sl1_loss_bwd(const float* const* pred, const float* const* gt,
                                   const uint8_t* const* mask, const int* hw, int B, int levels,
                                   const long long* counts, const float* grad_loss,
                                   float* const* grad_pred, void* stream) {
  LossLevels L;
  CASMVS_REQUIRE(grad_pred && counts && grad_loss, "sl1_loss_bwd: null pointer");
  if (int rc = make_levels(L, pred, gt, mask, grad_pred, hw, B, levels, "sl1_loss_bwd")) return rc;
  const long long total = L.begin[levels];
  sl1_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(L, counts, grad_loss);
  return after_launch("sl1_loss_bwd");
}
