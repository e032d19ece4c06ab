// Input pipeline, device side (SURVEY.md 8 f-4): uint8 RGB images -> normalised planar fp32.
//
// Replaces T.ToTensor() + T.Normalize(mean, std) of the reference's data sets
// (datasets/dtu.py:130-137) for images that are uploaded as BYTES: (N,H,W,3) uint8 ->
// (N,3,H,W) float32 with  y = ((float)x / 255 - mean[c]) / std[c]  in exactly that operation
// order (torchvision: .div(255), .sub_(mean), .div_(std)), so results are bit-identical to the
// host path while the H2D copy carries a quarter of the bytes.  HBM-bound: 3 B read + 12 B
// written per pixel; the 256 x 3 possible outputs are tabulated once per block.
//
// casmvs_jitter_normalize_u8_fwd puts the training split's T.ColorJitter(brightness, contrast)
// of the BlendedMVS reader (datasets/blendedmvs.py:130-137) in front of the same conversion,
// byte-exact to torchvision on PIL images: one integer luma-sum pass per image, then the
// normalise pass with each image's jitter folded into its table.
#include "common.cuh"

namespace casmvs {

// Writes image `ip` (hw RGB pixels) as three planes at `op` through the per-channel table `lut`.
// 4 pixels (12 bytes = 3 words) per thread per step when the planes of every image stay 16 B
// aligned (hw % 4 == 0); otherwise (N == 1, odd sizes) block 0's scalar path does everything.
__device__ __forceinline__ void lut_to_planes(const float (*lut)[256], const uint8_t* __restrict__ ip,
                                              float* __restrict__ op, size_t hw) {
  const size_t quads = (hw % 4 == 0) ? hw / 4 : 0;
  for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < quads;
       q += (size_t)gridDim.x * blockDim.x) {
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(ip + q * 12);
    const uint32_t a = __ldg(wp), b = __ldg(wp + 1), c = __ldg(wp + 2);
    // bytes: r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
    float4 r, g, bl;
    r.x = lut[0][a & 255];          g.x = lut[1][(a >> 8) & 255];   bl.x = lut[2][(a >> 16) & 255];
    r.y = lut[0][a >> 24];          g.y = lut[1][b & 255];          bl.y = lut[2][(b >> 8) & 255];
    r.z = lut[0][(b >> 16) & 255];  g.z = lut[1][b >> 24];          bl.z = lut[2][c & 255];
    r.w = lut[0][(c >> 8) & 255];   g.w = lut[1][(c >> 16) & 255];  bl.w = lut[2][c >> 24];
    st4(op + q * 4, r);
    st4(op + hw + q * 4, g);
    st4(op + 2 * hw + q * 4, bl);
  }
  if (blockIdx.x == 0) {
    for (size_t p = quads * 4 + threadIdx.x; p < hw; p += blockDim.x)
      for (int c = 0; c < 3; ++c) op[c * hw + p] = lut[c][ip[p * 3 + c]];
  }
}

__device__ __forceinline__ float normalize_value(int v, float mean, float sd) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), mean), sd);
}

__global__ void __launch_bounds__(256)
normalize_u8_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, size_t hw,
                    float m0, float m1, float m2, float s0, float s1, float s2) {
  __shared__ float lut[3][256];
  for (int i = threadIdx.x; i < 768; i += blockDim.x) {
    const int c = i >> 8, v = i & 255;
    const float mean = c == 0 ? m0 : c == 1 ? m1 : m2, sd = c == 0 ? s0 : c == 1 ? s1 : s2;
    lut[c][v] = normalize_value(v, mean, sd);
  }
  __syncthreads();
  const size_t n = blockIdx.y;
  lut_to_planes(lut, in + n * hw * 3, out + n * hw * 3, hw);
}

// ---- ColorJitter(brightness, contrast) on PIL images, then ToTensor + Normalize
//
// Pillow's Image.blend(im1, im2, alpha) per byte (libImaging/Blend.c):
//   t = (float)in1 + alpha * (float)(in2 - in1)   in float32, no FMA;
//   0 <= alpha <= 1: truncated to uint8; otherwise clamped to [0, 255], then truncated.
// Brightness is blend(black, img, b); contrast is blend(gray(m), img, c) where m is the mean of
// the image's L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16 rounded as int(mean + 0.5).  Both
// act on every byte alike, so the jitter of one image is a 256-entry byte table; only m needs a
// pass over the pixels (over the brightened image when brightness comes first).
__device__ __forceinline__ int pil_blend(int in1, int in2, float alpha) {
  const float t = __fadd_rn((float)in1, __fmul_rn(alpha, (float)(in2 - in1)));
  if (alpha >= 0.f && alpha <= 1.f) return (int)t;
  return t <= 0.f ? 0 : t >= 255.f ? 255 : (int)t;
}

__device__ __forceinline__ uint32_t pil_luma(uint32_t r, uint32_t g, uint32_t b) {
  return (r * 19595u + g * 38470u + b * 7471u + 0x8000u) >> 16;
}

// Pass 1: lsum[n] += sum of L over image n (brightened first when jitter[n*3] != 0).  Integer
// atomics keep the sum independent of the block order.
__global__ void __launch_bounds__(256)
jitter_luma_sum_kernel(const uint8_t* __restrict__ in, const float* __restrict__ jitter,
                       unsigned long long* __restrict__ lsum, size_t hw) {
  __shared__ uint32_t bt[256];
  __shared__ unsigned long long warp_sums[8];
  const size_t n = blockIdx.y;
  const bool bright_first = jitter[n * 3] != 0.f;
  const float b = jitter[n * 3 + 1];
  for (int v = threadIdx.x; v < 256; v += blockDim.x) bt[v] = bright_first ? pil_blend(0, v, b) : v;
  __syncthreads();
  const uint8_t* ip = in + n * hw * 3;
  uint32_t acc = 0;             // <= 255 per pixel; a thread sees far fewer than 2^24 pixels
  const size_t quads = (hw % 4 == 0) ? hw / 4 : 0;
  for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < quads;
       q += (size_t)gridDim.x * blockDim.x) {
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(ip + q * 12);
    const uint32_t a = __ldg(wp), w1 = __ldg(wp + 1), c = __ldg(wp + 2);
    acc += pil_luma(bt[a & 255], bt[(a >> 8) & 255], bt[(a >> 16) & 255]);
    acc += pil_luma(bt[a >> 24], bt[w1 & 255], bt[(w1 >> 8) & 255]);
    acc += pil_luma(bt[(w1 >> 16) & 255], bt[w1 >> 24], bt[c & 255]);
    acc += pil_luma(bt[(c >> 8) & 255], bt[(c >> 16) & 255], bt[c >> 24]);
  }
  if (blockIdx.x == 0) {
    for (size_t p = quads * 4 + threadIdx.x; p < hw; p += blockDim.x)
      acc += pil_luma(bt[ip[p * 3]], bt[ip[p * 3 + 1]], bt[ip[p * 3 + 2]]);
  }
  unsigned long long s = acc;
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += warp_sums[w];
    if (t) atomicAdd(lsum + n, t);
  }
}

// Pass 2: the jitter table of image n composed with the normalise table, then the planar store.
__global__ void __launch_bounds__(256)
jitter_normalize_u8_kernel(const uint8_t* __restrict__ in, const float* __restrict__ jitter,
                           const unsigned long long* __restrict__ lsum, float* __restrict__ out,
                           size_t hw, float m0, float m1, float m2, float s0, float s1, float s2) {
  __shared__ float lut[3][256];
  const size_t n = blockIdx.y;
  const bool bright_first = jitter[n * 3] != 0.f;
  const float b = jitter[n * 3 + 1], c = jitter[n * 3 + 2];
  // ImageStat's mean is sum / count in double; ImageEnhance.Contrast takes int(mean + 0.5)
  const int m = (int)(__ddiv_rn((double)lsum[n], (double)hw) + 0.5);
  for (int i = threadIdx.x; i < 768; i += blockDim.x) {
    const int ch = i >> 8, v = i & 255;
    const int y = bright_first ? pil_blend(m, pil_blend(0, v, b), c) : pil_blend(0, pil_blend(m, v, c), b);
    const float mean = ch == 0 ? m0 : ch == 1 ? m1 : m2, sd = ch == 0 ? s0 : ch == 1 ? s1 : s2;
    lut[ch][v] = normalize_value(y, mean, sd);
  }
  __syncthreads();
  lut_to_planes(lut, in + n * hw * 3, out + n * hw * 3, hw);
}

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_normalize_u8_fwd(const uint8_t* images, float* out, int N, int H, int W,
                                       const float* mean3, const float* std3, void* stream) {
  CASMVS_REQUIRE(images && out && mean3 && std3, "normalize_u8: null pointer");
  CASMVS_REQUIRE(N >= 0 && N <= 65535 && H > 0 && W > 0, "normalize_u8: bad dims");
  CASMVS_REQUIRE(std3[0] != 0.f && std3[1] != 0.f && std3[2] != 0.f, "normalize_u8: zero std");
  if (N == 0) return 0;
  const size_t hw = (size_t)H * W;
  // word loads / float4 stores need hw % 4 == 0 for every image after the first; otherwise
  // (never the case for the reference's 32-divisible image sizes) fall to one image per launch
  CASMVS_REQUIRE(hw % 4 == 0 || N == 1, "normalize_u8: H*W must be a multiple of 4 for N > 1");
  CASMVS_REQUIRE((reinterpret_cast<uintptr_t>(images) & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(out) & 15) == 0, "normalize_u8: misaligned");
  const unsigned bx = (unsigned)((hw / 4 + 255) / 256 < 1 ? 1 : (hw / 4 + 255) / 256);
  dim3 grd(bx < 2048 ? bx : 2048, (unsigned)N);
  normalize_u8_kernel<<<grd, 256, 0, as_stream(stream)>>>(images, out, hw, mean3[0], mean3[1],
                                                          mean3[2], std3[0], std3[1], std3[2]);
  return after_launch("normalize_u8");
}

extern "C" int casmvs_jitter_normalize_u8_fwd(const uint8_t* images, const float* jitter,
                                              float* out, long long* lsum, int N, int H, int W,
                                              const float* mean3, const float* std3, void* stream) {
  CASMVS_REQUIRE(images && jitter && out && lsum && mean3 && std3, "jitter_normalize_u8: null pointer");
  CASMVS_REQUIRE(N >= 0 && N <= 65535 && H > 0 && W > 0, "jitter_normalize_u8: bad dims");
  CASMVS_REQUIRE(std3[0] != 0.f && std3[1] != 0.f && std3[2] != 0.f, "jitter_normalize_u8: zero std");
  if (N == 0) return 0;
  const size_t hw = (size_t)H * W;
  CASMVS_REQUIRE(hw % 4 == 0 || N == 1, "jitter_normalize_u8: H*W must be a multiple of 4 for N > 1");
  CASMVS_REQUIRE(hw <= (1u << 31), "jitter_normalize_u8: more than 2^31 pixels per image");
  CASMVS_REQUIRE((reinterpret_cast<uintptr_t>(images) & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(jitter) & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(lsum) & 7) == 0, "jitter_normalize_u8: misaligned");
  cudaStream_t st = as_stream(stream);
  const cudaError_t e = cudaMemsetAsync(lsum, 0, (size_t)N * sizeof(long long), st);
  CASMVS_REQUIRE(e == cudaSuccess, "jitter_normalize_u8: memset failed: %s", cudaGetErrorString(e));
  const unsigned bx = (unsigned)((hw / 4 + 255) / 256 < 1 ? 1 : (hw / 4 + 255) / 256);
  dim3 grd(bx < 2048 ? bx : 2048, (unsigned)N);
  unsigned long long* sums = reinterpret_cast<unsigned long long*>(lsum);
  jitter_luma_sum_kernel<<<grd, 256, 0, st>>>(images, jitter, sums, hw);
  const int rc = after_launch("jitter_normalize_u8/luma_sum");
  if (rc) return rc;
  jitter_normalize_u8_kernel<<<grd, 256, 0, st>>>(images, jitter, sums, out, hw, mean3[0], mean3[1],
                                                  mean3[2], std3[0], std3[1], std3[2]);
  return after_launch("jitter_normalize_u8");
}
