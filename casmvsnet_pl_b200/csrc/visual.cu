// Training panels, device side: the reference image, depth_gt, depth_pred * mask and
// confidence * mask as one uint8 (H, n*W, 3) strip, the bytes TensorBoard stores for the original
// project's add_images('*/image_GT_pred_prob', stack) (train.py:107-114, :136-143), with the
// panels side by side and no padding.  A NULL input drops its panel; the remaining ones are
// packed left to right in that order, which gives visualize_depth / visualize_prob alone.
//
// Per pixel, with every step rounded as the host chain rounds it (explicit intrinsics, so
// nothing is contracted into an FMA; oracle/visual_oracle.py is the numpy restatement):
//
//   image   c = x / (1/s) after x - (-m/s), both constants float32 (torchvision Normalize),
//           then TensorBoard's u8((c * 255).clip(0, 255))
//   depth   v = nan_to_num(d) (NaN -> 0, +-inf -> +-FLT_MAX); mi = min of v over v > 0,
//           ma = max of v; g = u8(255 * ((v - mi) / (ma - mi + 1e-8f)));  colour JET[g]
//           (utils/visualization.py visualize_depth).  No v > 0: every pixel gets JET[0]; the
//           original raises there (np.min of an empty array).
//   prob    g = u8(255 * (p * m)); colour BONE[g] (visualize_prob)
//
// u8() is numpy's float32 -> uint8 cast on x86-64: truncate to int32 and keep the low byte; a
// value outside [-2^31, 2^31) and NaN become INT_MIN, byte 0.  So no clamp: -212.7 -> 44.
// The colour maps are cv2's, in cv2's BGR order written as RGB (the original passes cv2's BGR
// to Image.fromarray), and the ToTensor / TensorBoard round trip u8 / 255 * 255 is exact.
//
// Two launches: per-block partial (min positive, max) of both depth maps into the workspace,
// then every block folds the partials itself (min and max do not depend on order, so the
// result is deterministic) and draws its pixels.  Without a depth panel only the second runs.
#include <float.h>

#include "colormap_table.h"
#include "common.cuh"

namespace casmvs {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxPartials = CASMVS_VISUAL_WORKSPACE_BYTES / (4 * sizeof(float));

__device__ __forceinline__ uint8_t np_u8(float t) {
  return (t >= -2147483648.f && t < 2147483648.f) ? (uint8_t)__float2int_rz(t) : (uint8_t)0;
}

__device__ __forceinline__ float nan_to_num(float v) {
  return isnan(v) ? 0.f : isinf(v) ? (v > 0.f ? FLT_MAX : -FLT_MAX) : v;
}

__device__ __forceinline__ float masked(float v, const uint8_t* __restrict__ mask, size_t i) {
  return mask ? __fmul_rn(v, __ldg(mask + i) ? 1.f : 0.f) : v;
}

struct VisualArgs {
  const float *img, *gt, *pred, *conf;
  const uint8_t* mask;
  float* partials;           // (n_partials, 4): min positive gt, max gt, min positive pred, max pred
  uint8_t* out;
  int H, W, n_partials, n_panels;
};

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Reduces r[0..3] (min, max, min, max) over the block; thread 0 holds the result.
__device__ __forceinline__ void block_minmax(float (&r)[4]) {
  __shared__ float s[kThreads / 32][4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) r[k] = (k & 1) ? warp_max(r[k]) : warp_min(r[k]);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) s[warp][k] = r[k];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float v = lane < kThreads / 32 ? s[lane][k] : ((k & 1) ? -INFINITY : INFINITY);
      r[k] = (k & 1) ? warp_max(v) : warp_min(v);
    }
  }
}

__device__ __forceinline__ void fold(float (&r)[4], float v, int k) {
  if (v > 0.f) r[k] = fminf(r[k], v);
  r[k + 1] = fmaxf(r[k + 1], v);
}

__global__ void __launch_bounds__(kThreads) visual_minmax_kernel(const VisualArgs a) {
  const size_t npix = (size_t)a.H * a.W;
  float r[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < npix;
       i += (size_t)gridDim.x * kThreads) {
    if (a.gt) fold(r, nan_to_num(__ldg(a.gt + i)), 0);
    if (a.pred) fold(r, nan_to_num(masked(__ldg(a.pred + i), a.mask, i)), 2);
  }
  block_minmax(r);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) a.partials[blockIdx.x * 4 + k] = r[k];
  }
}

__device__ __forceinline__ void put(uint8_t* o, const uint8_t (&lut)[256][3], uint8_t g) {
  o[0] = lut[g][0];
  o[1] = lut[g][1];
  o[2] = lut[g][2];
}

// One depth panel pixel; mi = +inf when the map has no positive value.
__device__ __forceinline__ void depth_pixel(uint8_t* o, const uint8_t (&jet)[256][3], float v,
                                            float mi, float ma) {
  uint8_t g = 0;
  if (mi <= FLT_MAX) {
    const float den = __fadd_rn(__fsub_rn(ma, mi), 1e-8f);
    g = np_u8(__fmul_rn(255.f, __fdiv_rn(__fsub_rn(v, mi), den)));
  }
  put(o, jet, g);
}

__global__ void __launch_bounds__(kThreads) visual_draw_kernel(const VisualArgs a) {
  __shared__ uint8_t jet[256][3], bone[256][3];
  for (int t = threadIdx.x; t < 256 * 3; t += kThreads) {
    (&jet[0][0])[t] = (&kColormapJet[0][0])[t];
    (&bone[0][0])[t] = (&kColormapBone[0][0])[t];
  }
  float r[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
  if (a.gt || a.pred) {
    for (int p = threadIdx.x; p < a.n_partials; p += kThreads) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float v = a.partials[p * 4 + k];
        r[k] = (k & 1) ? fmaxf(r[k], v) : fminf(r[k], v);
      }
    }
    block_minmax(r);
  }
  __shared__ float range[4];
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) range[k] = r[k];
  }
  __syncthreads();
  // torchvision Normalize(mean=-m/s, std=1/s) with the ImageNet m, s (train.py:33-34)
  const float mean[3] = {(float)(-0.485 / 0.229), (float)(-0.456 / 0.224), (float)(-0.406 / 0.225)};
  const float stdv[3] = {(float)(1.0 / 0.229), (float)(1.0 / 0.224), (float)(1.0 / 0.225)};
  const size_t npix = (size_t)a.H * a.W;
  const size_t row = (size_t)a.n_panels * a.W * 3;
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < npix;
       i += (size_t)gridDim.x * kThreads) {
    const size_t y = i / a.W, x = i - y * a.W;
    uint8_t* o = a.out + y * row + x * 3;
    if (a.img) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = __fdiv_rn(__fsub_rn(__ldg(a.img + c * npix + i), mean[c]), stdv[c]);
        // numpy's clip keeps NaN and the cast makes it 0; fmaxf makes it 0 first
        o[c] = np_u8(fminf(fmaxf(__fmul_rn(v, 255.f), 0.f), 255.f));
      }
      o += (size_t)a.W * 3;
    }
    if (a.gt) {
      depth_pixel(o, jet, nan_to_num(__ldg(a.gt + i)), range[0], range[1]);
      o += (size_t)a.W * 3;
    }
    if (a.pred) {
      depth_pixel(o, jet, nan_to_num(masked(__ldg(a.pred + i), a.mask, i)), range[2], range[3]);
      o += (size_t)a.W * 3;
    }
    if (a.conf) put(o, bone, np_u8(__fmul_rn(255.f, masked(__ldg(a.conf + i), a.mask, i))));
  }
}

unsigned grid_for_pixels(size_t npix, int cap) {
  const size_t b = (npix + kThreads - 1) / kThreads;
  return (unsigned)(b < (size_t)cap ? b : cap);
}

}  // namespace

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_visual_panels(const float* img, const float* depth_gt,
                                    const float* depth_pred, const float* conf,
                                    const unsigned char* mask, int H, int W, unsigned char* out,
                                    void* workspace, void* stream) {
  CASMVS_REQUIRE(H > 0 && W > 0 && (size_t)H * W < (1ull << 31),
                 "visual_panels: bad dims H=%d W=%d", H, W);
  const int n_panels = !!img + !!depth_gt + !!depth_pred + !!conf;
  CASMVS_REQUIRE(n_panels > 0, "visual_panels: no panel input");
  CASMVS_REQUIRE(out, "visual_panels: null output");
  CASMVS_REQUIRE_ALIGNED("visual_panels", workspace, 16);
  CASMVS_REQUIRE(workspace || !(depth_gt || depth_pred), "visual_panels: null workspace");
  const size_t npix = (size_t)H * W;
  VisualArgs a{img, depth_gt, depth_pred, conf, mask, static_cast<float*>(workspace), out,
               H, W, (int)grid_for_pixels(npix, kMaxPartials), n_panels};
  cudaStream_t st = as_stream(stream);
  if (depth_gt || depth_pred) {
    visual_minmax_kernel<<<a.n_partials, kThreads, 0, st>>>(a);
    if (int rc = after_launch("visual_minmax")) return rc;
  }
  visual_draw_kernel<<<grid_for_pixels(npix, num_sms() * 8), kThreads, 0, st>>>(a);
  return after_launch("visual_draw");
}
