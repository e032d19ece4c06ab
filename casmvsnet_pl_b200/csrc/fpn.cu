// FeatureNet top-down path, fused (SURVEY.md §8f-2, first step): one kernel per pyramid level
//   feat = up2_bilinear(prev) + conv1x1(c; lat_w) + lat_b        (32 channels, never stored
//   out  = conv3x3(feat; smooth_w) + smooth_b                     for the finest level)
// Replaces (reference, relative to /root/reference) FeatureNet._upsample_add + lat{0,1} +
// smooth{0,1}, models/mvsnet.py:36-52: F.interpolate(x2, bilinear, align_corners=True),
// three elementwise passes and two cuDNN convolutions over a 32-channel full-resolution
// tensor (~750 MB of HBM traffic at 640x512x3 views) become ~100 MB.
// All tensors channels-last fp32; fp32 FMA arithmetic.
#include "common.cuh"

namespace casmvs {

constexpr int kFpnTile = 16;
constexpr int kFpnHalo = kFpnTile + 2;
constexpr int kFpnPix = 36;           // padded pixel pitch (floats) of the smem feature tile
constexpr int kFpnC = 32;             // pyramid width

template <int COUT>
__global__ void __launch_bounds__(256)
fpn_level_kernel(const float* __restrict__ prev,   // (N, h/2, w/2, 32)
                 const float* __restrict__ c,      // (N, h, w, CLAT)
                 const float* __restrict__ lat_w,  // (32, CLAT)
                 const float* __restrict__ lat_b,  // (32)
                 const float* __restrict__ sm_w,   // (COUT, 32, 3, 3)
                 const float* __restrict__ sm_b,   // (COUT)
                 float* __restrict__ feat_out,     // (N, h, w, 32) or null
                 float* __restrict__ out,          // (N, h, w, COUT)
                 int h, int w, int CLAT) {
  extern __shared__ __align__(16) float smem[];
  float* s_feat = smem;                                   // [18*18][36]
  float* s_smw = s_feat + kFpnHalo * kFpnHalo * kFpnPix;  // [9][32][COUT]
  float* s_latw = s_smw + 9 * kFpnC * COUT;               // [CLAT][32]
  const int n = blockIdx.z;
  const int y0 = blockIdx.y * kFpnTile, x0 = blockIdx.x * kFpnTile;
  const int hi = h / 2, wi = w / 2;

  for (int i = threadIdx.x; i < 9 * kFpnC * COUT; i += blockDim.x) {
    const int co = i % COUT, ci = (i / COUT) % kFpnC, tap = i / (COUT * kFpnC);
    s_smw[i] = __ldg(sm_w + ((size_t)co * kFpnC + ci) * 9 + tap);
  }
  for (int i = threadIdx.x; i < CLAT * kFpnC; i += blockDim.x) {
    const int ch = i % kFpnC, ci = i / kFpnC;
    s_latw[i] = __ldg(lat_w + (size_t)ch * CLAT + ci);
  }
  __syncthreads();

  // ---- phase 1: the 18x18 halo'd feature tile, 8 channels per work item ----
  const float sy = hi > 1 ? (float)(hi - 1) / (float)(h - 1) : 0.f;
  const float sx = wi > 1 ? (float)(wi - 1) / (float)(w - 1) : 0.f;
  const float* pn = prev + (size_t)n * hi * wi * kFpnC;
  const float* cn = c + (size_t)n * h * w * CLAT;
  for (int it = threadIdx.x; it < kFpnHalo * kFpnHalo * 4; it += blockDim.x) {
    const int g = it & 3, hp = it >> 2;
    const int ty = hp / kFpnHalo, tx = hp - ty * kFpnHalo;
    const int y = y0 - 1 + ty, x = x0 - 1 + tx;
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = 0.f;
    if (y >= 0 && y < h && x >= 0 && x < w) {               // outside the image: zero padding
      const float fy = sy * (float)y, fx = sx * (float)x;
      int ya = min((int)fy, hi - 1), xa = min((int)fx, wi - 1);
      const int yb = min(ya + 1, hi - 1), xb = min(xa + 1, wi - 1);
      const float ly = fy - (float)ya, lx = fx - (float)xa;
      const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx),
                  w11 = ly * lx;
      const float* p00 = pn + ((size_t)ya * wi + xa) * kFpnC + g * 8;
      const float* p01 = pn + ((size_t)ya * wi + xb) * kFpnC + g * 8;
      const float* p10 = pn + ((size_t)yb * wi + xa) * kFpnC + g * 8;
      const float* p11 = pn + ((size_t)yb * wi + xb) * kFpnC + g * 8;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float4 a = ldg4(p00 + 4 * q), b = ldg4(p01 + 4 * q), cc = ldg4(p10 + 4 * q),
                     d = ldg4(p11 + 4 * q);
        v[4 * q + 0] = a.x * w00 + b.x * w01 + cc.x * w10 + d.x * w11;
        v[4 * q + 1] = a.y * w00 + b.y * w01 + cc.y * w10 + d.y * w11;
        v[4 * q + 2] = a.z * w00 + b.z * w01 + cc.z * w10 + d.z * w11;
        v[4 * q + 3] = a.w * w00 + b.w * w01 + cc.w * w10 + d.w * w11;
      }
      const float* cp = cn + ((size_t)y * w + x) * CLAT;
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] += __ldg(lat_b + g * 8 + k);
      for (int ci = 0; ci < CLAT; ci += 4) {
        const float4 cv = ldg4(cp + ci);
        const float cs[4] = {cv.x, cv.y, cv.z, cv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float* wr = s_latw + (ci + j) * kFpnC + g * 8;
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] = fmaf(cs[j], wr[k], v[k]);
        }
      }
      if (feat_out && ty >= 1 && ty <= kFpnTile && tx >= 1 && tx <= kFpnTile) {
        float* fo = feat_out + (((size_t)n * h + y) * w + x) * kFpnC + g * 8;
        st4(fo, make_float4(v[0], v[1], v[2], v[3]));
        st4(fo + 4, make_float4(v[4], v[5], v[6], v[7]));
      }
    }
    float* sp = s_feat + hp * kFpnPix + g * 8;
    *reinterpret_cast<float4*>(sp) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(sp + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
  __syncthreads();

  // ---- phase 2: 3x3 smoothing conv, one output pixel per thread ----
  const int ty = threadIdx.x / kFpnTile, tx = threadIdx.x % kFpnTile;
  const int y = y0 + ty, x = x0 + tx;
  float acc[COUT];
#pragma unroll
  for (int k = 0; k < COUT; ++k) acc[k] = __ldg(sm_b + k);
#pragma unroll
  for (int dy = 0; dy < 3; ++dy) {
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const float* fp = s_feat + ((ty + dy) * kFpnHalo + tx + dx) * kFpnPix;
      const float* wp = s_smw + (dy * 3 + dx) * kFpnC * COUT;
#pragma unroll
      for (int ci = 0; ci < kFpnC; ci += 4) {
        const float4 f = *reinterpret_cast<const float4*>(fp + ci);
        const float fs[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
          for (int k = 0; k < COUT; k += 4) {
            const float4 wv = *reinterpret_cast<const float4*>(wp + (ci + j) * COUT + k);
            acc[k] = fmaf(fs[j], wv.x, acc[k]);
            acc[k + 1] = fmaf(fs[j], wv.y, acc[k + 1]);
            acc[k + 2] = fmaf(fs[j], wv.z, acc[k + 2]);
            acc[k + 3] = fmaf(fs[j], wv.w, acc[k + 3]);
          }
        }
      }
    }
  }
  if (y < h && x < w) {
    float* op = out + (((size_t)n * h + y) * w + x) * COUT;
#pragma unroll
    for (int k = 0; k < COUT; k += 4) st4(op + k, make_float4(acc[k], acc[k + 1], acc[k + 2], acc[k + 3]));
  }
}

__device__ __forceinline__ float round_tf32_if(float x, int on) {
  if (!on) return x;
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// feat[n,y,x,:] = up2_bilinear(prev)[n,y,x,:] + lat_w @ c[n,y,x,:] + lat_b  (32 channels).
// Four threads per pixel (8 channels each) x kMergeP pixels per thread.  The kernel is bound
// by the L1/shared pipe with one pixel per thread:
// every 128-bit shared or global access costs a warp four L1 cycles, so the lateral weights
// of a channel group are read from shared memory once per kMergeP pixels instead of once per
// pixel.  HBM traffic: reads c + prev (a quarter of the pixels), writes 128 B per pixel.
constexpr int kMergeP = 4;
__global__ void __launch_bounds__(256)
fpn_merge_kernel(const float* __restrict__ prev,   // (N, h/2, w/2, 32) or null
                 const float* __restrict__ c,      // (N, h, w, CLAT)
                 const float* __restrict__ lat_w,  // (32, CLAT)
                 const float* __restrict__ lat_b,  // (32)
                 float* __restrict__ feat,         // (N, h, w, 32)
                 int N, int h, int w, int CLAT, int round_out) {
  extern __shared__ __align__(16) float s_latw[];   // [CLAT][32] + bias [32]
  for (int i = threadIdx.x; i < CLAT * kFpnC; i += blockDim.x) {
    const int ch = i % kFpnC, ci = i / kFpnC;
    s_latw[i] = __ldg(lat_w + (size_t)ch * CLAT + ci);
  }
  for (int i = threadIdx.x; i < kFpnC; i += blockDim.x) s_latw[CLAT * kFpnC + i] = __ldg(lat_b + i);
  __syncthreads();
  const int hi = h / 2, wi = w / 2;
  const float sy = hi > 1 ? (float)(hi - 1) / (float)(h - 1) : 0.f;
  const float sx = wi > 1 ? (float)(wi - 1) / (float)(w - 1) : 0.f;
  const int n = blockIdx.y;
  const int g = threadIdx.x & 3;
  const int hw = h * w;
  // pixels of this thread: p0 + k*64 (a block covers 64*kMergeP consecutive pixels of image n)
  const int p0 = blockIdx.x * (64 * kMergeP) + (threadIdx.x >> 2);
  float v[kMergeP][8];
#pragma unroll
  for (int k = 0; k < kMergeP; ++k) {
    const int pix = p0 + k * 64;
#pragma unroll
    for (int q = 0; q < 8; ++q) v[k][q] = s_latw[CLAT * kFpnC + g * 8 + q];
    if (prev && pix < hw) {
      const int y = pix / w, x = pix - y * w;
      const float* pn = prev + (size_t)n * hi * wi * kFpnC;
      const float fy = sy * (float)y, fx = sx * (float)x;
      const int ya = min((int)fy, hi - 1), xa = min((int)fx, wi - 1);
      const int yb = min(ya + 1, hi - 1), xb = min(xa + 1, wi - 1);
      const float ly = fy - (float)ya, lx = fx - (float)xa;
      const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx),
                  w11 = ly * lx;
      const float* p00 = pn + ((size_t)ya * wi + xa) * kFpnC + g * 8;
      const float* p01 = pn + ((size_t)ya * wi + xb) * kFpnC + g * 8;
      const float* p10 = pn + ((size_t)yb * wi + xa) * kFpnC + g * 8;
      const float* p11 = pn + ((size_t)yb * wi + xb) * kFpnC + g * 8;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float4 a = ldg4(p00 + 4 * q), b = ldg4(p01 + 4 * q), cc = ldg4(p10 + 4 * q),
                     d = ldg4(p11 + 4 * q);
        // same association as the fused level kernel: ((a*w00 + b*w01) + c*w10) + d*w11, then + bias
        v[k][4 * q + 0] = (a.x * w00 + b.x * w01 + cc.x * w10 + d.x * w11) + v[k][4 * q + 0];
        v[k][4 * q + 1] = (a.y * w00 + b.y * w01 + cc.y * w10 + d.y * w11) + v[k][4 * q + 1];
        v[k][4 * q + 2] = (a.z * w00 + b.z * w01 + cc.z * w10 + d.z * w11) + v[k][4 * q + 2];
        v[k][4 * q + 3] = (a.w * w00 + b.w * w01 + cc.w * w10 + d.w * w11) + v[k][4 * q + 3];
      }
    }
  }
  const float* cn = c + (size_t)n * hw * CLAT;
  for (int ci = 0; ci < CLAT; ci += 4) {
    float cs[kMergeP][4];
#pragma unroll
    for (int k = 0; k < kMergeP; ++k) {
      const int pix = p0 + k * 64;
      const float4 cv = pix < hw ? ldg4(cn + (size_t)pix * CLAT + ci) : make_float4(0.f, 0.f, 0.f, 0.f);
      cs[k][0] = cv.x; cs[k][1] = cv.y; cs[k][2] = cv.z; cs[k][3] = cv.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 wa = *reinterpret_cast<const float4*>(s_latw + (ci + j) * kFpnC + g * 8);
      const float4 wb = *reinterpret_cast<const float4*>(s_latw + (ci + j) * kFpnC + g * 8 + 4);
      const float wr[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
      for (int k = 0; k < kMergeP; ++k) {
#pragma unroll
        for (int q = 0; q < 8; ++q) v[k][q] = fmaf(cs[k][j], wr[q], v[k][q]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kMergeP; ++k) {
    const int pix = p0 + k * 64;
    if (pix < hw) {
#pragma unroll
      for (int q = 0; q < 8; ++q) v[k][q] = round_tf32_if(v[k][q], round_out);
      float* fo = feat + ((size_t)n * hw + pix) * kFpnC + g * 8;
      st4(fo, make_float4(v[k][0], v[k][1], v[k][2], v[k][3]));
      st4(fo + 4, make_float4(v[k][4], v[k][5], v[k][6], v[k][7]));
    }
  }
}

// y[n,y,x,0:8] = lrelu(conv3x3(x[n,0:3], w) + bias): planar RGB in, channels-last out.
// One output pixel per thread; the 3x3x3 neighbourhood comes through L1 (threads of a warp
// are consecutive in x, so every plane row is read coalesced); weights [27][8] in smem.
__global__ void __launch_bounds__(256)
conv2d_rgb8_kernel(const float* __restrict__ x, const float* __restrict__ w,
                   const float* __restrict__ bias, float slope, float* __restrict__ y, int N,
                   int H, int W, int round_out) {
  __shared__ __align__(16) float s_w[27 * 8 + 8];
  for (int i = threadIdx.x; i < 27 * 8; i += blockDim.x) {
    const int co = i & 7, r = i >> 3;            // r = ci*9 + ky*3 + kx  (torch (8,3,3,3) order)
    s_w[i] = __ldg(w + (size_t)co * 27 + r);
  }
  if (threadIdx.x < 8) s_w[27 * 8 + threadIdx.x] = __ldg(bias + threadIdx.x);
  __syncthreads();
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  const int py = blockIdx.y, n = blockIdx.z;
  if (px >= W) return;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = s_w[27 * 8 + k];
  const float* xn = x + (size_t)n * 3 * H * W;
#pragma unroll
  for (int ci = 0; ci < 3; ++ci) {
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = py + ky - 1;
      const bool yok = iy >= 0 && iy < H;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = px + kx - 1;
        const float v = (yok && ix >= 0 && ix < W) ? __ldg(xn + ((size_t)ci * H + iy) * W + ix) : 0.f;
        const float4 w0 = *reinterpret_cast<const float4*>(s_w + (ci * 9 + ky * 3 + kx) * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(s_w + (ci * 9 + ky * 3 + kx) * 8 + 4);
        acc[0] = fmaf(v, w0.x, acc[0]); acc[1] = fmaf(v, w0.y, acc[1]);
        acc[2] = fmaf(v, w0.z, acc[2]); acc[3] = fmaf(v, w0.w, acc[3]);
        acc[4] = fmaf(v, w1.x, acc[4]); acc[5] = fmaf(v, w1.y, acc[5]);
        acc[6] = fmaf(v, w1.z, acc[6]); acc[7] = fmaf(v, w1.w, acc[7]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float t = acc[k] >= 0.f ? acc[k] : acc[k] * slope;
    acc[k] = round_tf32_if(t, round_out);
  }
  float* yo = y + (((size_t)n * H + py) * W + px) * 8;
  st4(yo, make_float4(acc[0], acc[1], acc[2], acc[3]));
  st4(yo + 4, make_float4(acc[4], acc[5], acc[6], acc[7]));
}

// Same, four consecutive output pixels per thread (W % 4 == 0): each input row segment
// x-1 .. x+4 is loaded once (scalar, float4, scalar) and each tap's 8 weights are read from
// shared memory once for the four pixels -- about a third of the instructions per pixel.
__global__ void __launch_bounds__(256)
conv2d_rgb8_x4_kernel(const float* __restrict__ x, const float* __restrict__ w,
                      const float* __restrict__ bias, float slope, float* __restrict__ y, int N,
                      int H, int W, int round_out) {
  __shared__ __align__(16) float s_w[27 * 8 + 8];
  for (int i = threadIdx.x; i < 27 * 8; i += blockDim.x) {
    const int co = i & 7, r = i >> 3;            // r = ci*9 + ky*3 + kx  (torch (8,3,3,3) order)
    s_w[i] = __ldg(w + (size_t)co * 27 + r);
  }
  if (threadIdx.x < 8) s_w[27 * 8 + threadIdx.x] = __ldg(bias + threadIdx.x);
  __syncthreads();
  const int px = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int py = blockIdx.y, n = blockIdx.z;
  if (px >= W) return;
  float acc[4][8];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[p][k] = s_w[27 * 8 + k];
  const float* xn = x + (size_t)n * 3 * H * W;
#pragma unroll
  for (int ci = 0; ci < 3; ++ci) {
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = py + ky - 1;
      float in[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (iy >= 0 && iy < H) {
        const float* row = xn + ((size_t)ci * H + iy) * W + px;
        const float4 mid = ldg4(row);
        in[1] = mid.x; in[2] = mid.y; in[3] = mid.z; in[4] = mid.w;
        if (px > 0) in[0] = __ldg(row - 1);
        if (px + 4 < W) in[5] = __ldg(row + 4);
      }
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const float4 w0 = *reinterpret_cast<const float4*>(s_w + (ci * 9 + ky * 3 + kx) * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(s_w + (ci * 9 + ky * 3 + kx) * 8 + 4);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float v = in[p + kx];
          acc[p][0] = fmaf(v, w0.x, acc[p][0]); acc[p][1] = fmaf(v, w0.y, acc[p][1]);
          acc[p][2] = fmaf(v, w0.z, acc[p][2]); acc[p][3] = fmaf(v, w0.w, acc[p][3]);
          acc[p][4] = fmaf(v, w1.x, acc[p][4]); acc[p][5] = fmaf(v, w1.y, acc[p][5]);
          acc[p][6] = fmaf(v, w1.z, acc[p][6]); acc[p][7] = fmaf(v, w1.w, acc[p][7]);
        }
      }
    }
  }
  float* yo = y + (((size_t)n * H + py) * W + px) * 8;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float t = acc[p][k] >= 0.f ? acc[p][k] : acc[p][k] * slope;
      acc[p][k] = round_tf32_if(t, round_out);
    }
    st4(yo + p * 8, make_float4(acc[p][0], acc[p][1], acc[p][2], acc[p][3]));
    st4(yo + p * 8 + 4, make_float4(acc[p][4], acc[p][5], acc[p][6], acc[p][7]));
  }
}

// x[..., c] = lrelu(x[..., c] + bias[c]) in place on a channels-last tensor (C % 4 == 0):
// the tail of a folded conv+ABN block when the conv itself comes from cuDNN.
__global__ void __launch_bounds__(256)
bias_lrelu_kernel(float* __restrict__ x, const float* __restrict__ bias, float slope, size_t n4,
                  int C, int round_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int c = (int)((i * 4) % (size_t)C);
  float4 v = *reinterpret_cast<float4*>(x + i * 4);
  const float4 b = ldg4(bias + c);
  v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
  v.x = v.x >= 0.f ? v.x : v.x * slope; v.y = v.y >= 0.f ? v.y : v.y * slope;
  v.z = v.z >= 0.f ? v.z : v.z * slope; v.w = v.w >= 0.f ? v.w : v.w * slope;
  v.x = round_tf32_if(v.x, round_out); v.y = round_tf32_if(v.y, round_out);
  v.z = round_tf32_if(v.z, round_out); v.w = round_tf32_if(v.w, round_out);
  *reinterpret_cast<float4*>(x + i * 4) = v;
}

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_bias_act_nhwc(float* x, const float* bias, float slope, size_t numel,
                                    int C, int round_tf32, void* stream) {
  CASMVS_REQUIRE(x && bias, "bias_act: null pointer");
  CASMVS_REQUIRE(C > 0 && C % 4 == 0 && numel % (size_t)C == 0, "bias_act: C %% 4 != 0 or ragged");
  if (numel == 0) return 0;
  const size_t n4 = numel / 4;
  bias_lrelu_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, as_stream(stream)>>>(
      x, bias, slope, n4, C, round_tf32 ? 1 : 0);
  return after_launch("bias_act");
}

extern "C" int casmvs_bias_lrelu_nhwc(float* x, const float* bias, float slope, size_t numel,
                                      int C, void* stream) {
  return casmvs_bias_act_nhwc(x, bias, slope, numel, C, 0, stream);
}

extern "C" int casmvs_fpn_level_fwd(const float* prev, const float* c, const float* lat_w,
                                    const float* lat_b, const float* smooth_w,
                                    const float* smooth_b, float* feat_out, float* out, int N,
                                    int h, int w, int CLAT, int COUT, void* stream) {
  CASMVS_REQUIRE(prev && c && lat_w && lat_b && smooth_w && smooth_b && out, "fpn_level: null pointer");
  CASMVS_REQUIRE(N >= 0 && N <= 65535 && h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0,
                 "fpn_level: bad dims (h,w even, >= 2)");
  CASMVS_REQUIRE(CLAT % 4 == 0 && CLAT > 0 && CLAT <= 64, "fpn_level: CLAT must be a multiple of 4");
  CASMVS_REQUIRE(COUT == 8 || COUT == 16, "fpn_level: COUT must be 8 or 16 (got %d)", COUT);
  if (N == 0) return 0;
  dim3 grd((w + kFpnTile - 1) / kFpnTile, (h + kFpnTile - 1) / kFpnTile, N);
  const size_t smem = (size_t)(kFpnHalo * kFpnHalo * kFpnPix + 9 * kFpnC * COUT + CLAT * kFpnC) * 4;
  cudaStream_t st = as_stream(stream);
  if (COUT == 8) {
    static std::atomic<bool> a[kMaxDevices];
    if (int rc = opt_in_smem(fpn_level_kernel<8>, 100 * 1024, a, "fpn_level")) return rc;
    fpn_level_kernel<8><<<grd, 256, smem, st>>>(prev, c, lat_w, lat_b, smooth_w, smooth_b, feat_out, out, h, w, CLAT);
  } else {
    static std::atomic<bool> a[kMaxDevices];
    if (int rc = opt_in_smem(fpn_level_kernel<16>, 100 * 1024, a, "fpn_level")) return rc;
    fpn_level_kernel<16><<<grd, 256, smem, st>>>(prev, c, lat_w, lat_b, smooth_w, smooth_b, feat_out, out, h, w, CLAT);
  }
  return after_launch("fpn_level");
}

extern "C" int casmvs_fpn_merge_fwd(const float* prev, const float* c, const float* lat_w,
                                    const float* lat_b, float* feat, int N, int h, int w,
                                    int CLAT, int round_tf32, void* stream) {
  CASMVS_REQUIRE(c && lat_w && lat_b && feat, "fpn_merge: null pointer");
  CASMVS_REQUIRE(N >= 0 && h >= 1 && w >= 1, "fpn_merge: bad dims");
  CASMVS_REQUIRE(!prev || (h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0),
                 "fpn_merge: h,w must be even when a coarser level is upsampled");
  CASMVS_REQUIRE(CLAT % 4 == 0 && CLAT > 0 && CLAT <= 64, "fpn_merge: CLAT must be a multiple of 4");
  if (N == 0) return 0;
  CASMVS_REQUIRE(N <= 65535 && (long)h * w < (1l << 30), "fpn_merge: volume too large");
  const size_t smem = (size_t)(CLAT * kFpnC + kFpnC) * 4;
  dim3 blocks((h * w + 64 * kMergeP - 1) / (64 * kMergeP), N);
  fpn_merge_kernel<<<blocks, 256, smem, as_stream(stream)>>>(prev, c, lat_w, lat_b, feat, N, h, w,
                                                            CLAT, round_tf32 ? 1 : 0);
  return after_launch("fpn_merge");
}

extern "C" int casmvs_conv2d_rgb8_fwd(const float* x, const float* w, const float* bias,
                                      float slope, float* y, int N, int H, int W,
                                      int round_tf32, void* stream) {
  CASMVS_REQUIRE(x && w && bias && y, "conv2d_rgb8: null pointer");
  CASMVS_REQUIRE(N >= 0 && N <= 65535 && H >= 1 && H <= 65535 && W >= 1, "conv2d_rgb8: bad dims");
  if (N == 0) return 0;
  if (W % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const int bx = W / 4 >= 256 ? 256 : ((W / 4 + 31) / 32) * 32;     // one block per row up to 1024 px
    dim3 grd((W / 4 + bx - 1) / bx, H, N);
    conv2d_rgb8_x4_kernel<<<grd, bx, 0, as_stream(stream)>>>(x, w, bias, slope, y, N, H, W,
                                                             round_tf32 ? 1 : 0);
    return after_launch("conv2d_rgb8");
  }
  dim3 grd((W + 127) / 128, H, N);
  conv2d_rgb8_kernel<<<grd, 128, 0, as_stream(stream)>>>(x, w, bias, slope, y, N, H, W,
                                                         round_tf32 ? 1 : 0);
  return after_launch("conv2d_rgb8");
}

// ---- fp32 (CUDA-core) 5x5 stride-2 pad-2 convolution ---------------------------------------
// The fp32 precision mode of FeatureNet's two strided blocks (ConvBnReLU(8,16,5,2,2) /
// (16,32,5,2,2), mvsnet.py:16,20): bit-faithful products like every kernel of that mode.
// CTA = 16 x 8 output pixels x all COUT; the (35 x 19) input footprint is staged in shared
// memory planar per channel (stride-2 reads of neighbouring threads: 2-way bank conflict at
// worst), the weights [25][CIN][COUT] are read as warp broadcasts.
namespace casmvs {

template <int CIN, int COUT>
__global__ void __launch_bounds__(128)
conv2d_5x5s2_fp32_kernel(const float* __restrict__ x, const float* __restrict__ wt,
                         const float* __restrict__ shift, float slope, float* __restrict__ y,
                         int H, int W, int Ho, int Wo) {
  constexpr int TX = 16, TY = 8, IW = 2 * TX + 3, IH = 2 * TY + 3, IWP = IW + 1;
  extern __shared__ __align__(16) float s_raw[];
  float* s_in = s_raw;                          // [CIN][IH][IWP]
  float* s_w = s_raw + CIN * IH * IWP;          // [25][CIN][COUT]
  const int n = blockIdx.z;
  const int ox0 = blockIdx.x * TX, oy0 = blockIdx.y * TY;
  const int ix0 = 2 * ox0 - 2, iy0 = 2 * oy0 - 2;
  const float* xb = x + (size_t)n * H * W * CIN;
  for (int i = threadIdx.x; i < IH * IW * CIN; i += blockDim.x) {
    const int ci = i % CIN, xx = (i / CIN) % IW, yy = i / (CIN * IW);
    const int gx = ix0 + xx, gy = iy0 + yy;
    s_in[(ci * IH + yy) * IWP + xx] =
        (gx >= 0 && gx < W && gy >= 0 && gy < H) ? __ldg(xb + ((size_t)gy * W + gx) * CIN + ci) : 0.f;
  }
  for (int i = threadIdx.x; i < 25 * CIN * COUT; i += blockDim.x) {
    const int co = i % COUT, ci = (i / COUT) % CIN, tap = i / (COUT * CIN);
    s_w[i] = __ldg(wt + ((size_t)co * CIN + ci) * 25 + tap);      // torch (Cout,Cin,5,5)
  }
  __syncthreads();
  const int lx = threadIdx.x % TX, ly = threadIdx.x / TX;
  float acc[COUT];
#pragma unroll
  for (int k = 0; k < COUT; ++k) acc[k] = 0.f;
  for (int ky = 0; ky < 5; ++ky)
    for (int kx = 0; kx < 5; ++kx) {
      const float* wrow = s_w + (size_t)(ky * 5 + kx) * CIN * COUT;
#pragma unroll 4
      for (int ci = 0; ci < CIN; ++ci) {
        const float a = s_in[(ci * IH + 2 * ly + ky) * IWP + 2 * lx + kx];
#pragma unroll
        for (int k = 0; k < COUT; k += 4) {
          const float4 w4 = *reinterpret_cast<const float4*>(wrow + ci * COUT + k);
          acc[k] = fmaf(a, w4.x, acc[k]);         acc[k + 1] = fmaf(a, w4.y, acc[k + 1]);
          acc[k + 2] = fmaf(a, w4.z, acc[k + 2]); acc[k + 3] = fmaf(a, w4.w, acc[k + 3]);
        }
      }
    }
  const int ox = ox0 + lx, oy = oy0 + ly;
  if (ox >= Wo || oy >= Ho) return;
  float* op = y + (((size_t)n * Ho + oy) * Wo + ox) * COUT;
#pragma unroll
  for (int k = 0; k < COUT; k += 4) {
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float t = acc[k + j] + (shift ? __ldg(shift + k + j) : 0.f);
      v[j] = t >= 0.f ? t : t * slope;
    }
    st4(op + k, make_float4(v[0], v[1], v[2], v[3]));
  }
}

template <int CIN, int COUT>
static int launch_5x5_fp32(const float* x, const float* w, const float* shift, float slope, float* y,
                           int N, int H, int W, cudaStream_t st) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  constexpr int smem = (CIN * 19 * 36 + 25 * CIN * COUT) * 4;
  auto kfn = conv2d_5x5s2_fp32_kernel<CIN, COUT>;
  static std::atomic<bool> a[kMaxDevices];
  if (int rc = opt_in_smem(kfn, smem, a, "conv2d_5x5s2_fp32")) return rc;
  dim3 grd((Wo + 15) / 16, (Ho + 7) / 8, N);
  kfn<<<grd, 128, smem, st>>>(x, w, shift, slope, y, H, W, Ho, Wo);
  return after_launch("conv2d_5x5s2_fp32");
}

}  // namespace casmvs

extern "C" int casmvs_conv2d_5x5s2_fp32_fwd(const float* x, const float* w, const float* shift,
                                            float slope, float* y, int N, int Cin, int Cout,
                                            int H, int W, void* stream) {
  CASMVS_REQUIRE(x && w && y, "conv2d_5x5s2_fp32: null pointer");
  CASMVS_REQUIRE(N >= 0 && N <= 65535 && H >= 1 && W >= 1, "conv2d_5x5s2_fp32: bad dims");
  if (N == 0) return 0;
  cudaStream_t st = as_stream(stream);
  if (Cin == 8 && Cout == 16) return casmvs::launch_5x5_fp32<8, 16>(x, w, shift, slope, y, N, H, W, st);
  if (Cin == 16 && Cout == 32) return casmvs::launch_5x5_fp32<16, 32>(x, w, shift, slope, y, N, H, W, st);
  set_error("conv2d_5x5s2_fp32: only the FeatureNet shapes 8->16 and 16->32 are built (got %d->%d)",
            Cin, Cout);
  return -1;
}
