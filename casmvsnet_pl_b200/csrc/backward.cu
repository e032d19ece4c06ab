// Backward kernels of the hot path (SURVEY.md 8 f-1): what `loss.backward()` of the reference's
// training step (train.py:99-127, losses.py:10-17) needs from K1, K2 and K3.
//
//   casmvs_warp_cost_bwd   d(cost volume)/d(features): grid_sample's backward (bilinear
//                          scatter-add into the source features, models/modules.py:87-89)
//                          chained with the variance / group-wise-correlation reduction
//                          (models/mvsnet.py:147-172).  Hypotheses are detached
//                          (mvsnet.py:231) and projections are data: no other gradient exists.
//   casmvs_conv3d_wgrad    d/d(weight) of Conv3d / ConvTranspose3d (modules.py:26,
//                          mvsnet.py:75-89).  The data gradients need no kernel of their own:
//                          dgrad(conv s1) = conv s1 with flipped / transposed weights,
//                          dgrad(conv s2) = the transposed conv, dgrad(transposed) = conv s2 —
//                          all served by casmvs_conv3d_fwd.
//   casmvs_regress_bwd     d(depth)/d(logits) of softmax + expectation (mvsnet.py:174-177);
//                          the confidence branch is under no_grad in the reference (:179).
// fp32, CUDA cores, atomics for the scatter: correctness-first kernels (training at the
// reference's 640x512 crop is bandwidth-light next to inference at 1152x864).
#include "k1_common.cuh"

namespace casmvs {

struct TapPos { unsigned off; float w00, w01, w10, w11; };

// same arithmetic as gather_sample (k1_common.cuh): clamped 2x2 window + remapped weights
__device__ __forceinline__ TapPos tap_pos(float qx, float qy, float qz, int h, int w, int C) {
  const float rz = rcp_approx(qz);
  const float u = qx * rz, v = qy * rz;
  const float x0f = floorf(u), y0f = floorf(v);
  const int x0 = __float2int_rd(u), y0 = __float2int_rd(v);
  const bool valid = (qz > 1e-7f) && (unsigned)(x0 + 1) <= (unsigned)w &&
                     (unsigned)(y0 + 1) <= (unsigned)h;
  const float fx = u - x0f, fy = v - y0f;
  float wxa = 1.f - fx, wxb = fx, wya = 1.f - fy, wyb = fy;
  if (x0 < 0) { wxa = wxb; wxb = 0.f; }
  if (x0 > w - 2) { wxb = wxa; wxa = 0.f; }
  if (y0 < 0) { wya = wyb; wyb = 0.f; }
  if (y0 > h - 2) { wyb = wya; wya = 0.f; }
  if (!valid) { wxa = 0.f; wxb = 0.f; }
  const int xs = min(max(x0, 0), w - 2), ys = min(max(y0, 0), h - 2);
  TapPos t;
  t.w00 = wxa * wya; t.w01 = wxb * wya; t.w10 = wxa * wyb; t.w11 = wxb * wyb;
  t.off = (unsigned)((ys * w + xs) * C);
  return t;
}

__device__ __forceinline__ void blend8f(const float* __restrict__ p, int C, int row, const TapPos& t,
                                        float (&r)[8]) {
  const float4 a0 = ldg4(p), a1 = ldg4(p + 4), b0 = ldg4(p + C), b1 = ldg4(p + C + 4);
  const float4 c0 = ldg4(p + row), c1 = ldg4(p + row + 4), d0 = ldg4(p + row + C),
               d1 = ldg4(p + row + C + 4);
#define B8(i, A, Bq, Cq, Dq) r[i] = fmaf(Dq, t.w11, fmaf(Cq, t.w10, fmaf(Bq, t.w01, A * t.w00)));
  B8(0, a0.x, b0.x, c0.x, d0.x) B8(1, a0.y, b0.y, c0.y, d0.y) B8(2, a0.z, b0.z, c0.z, d0.z)
  B8(3, a0.w, b0.w, c0.w, d0.w) B8(4, a1.x, b1.x, c1.x, d1.x) B8(5, a1.y, b1.y, c1.y, d1.y)
  B8(6, a1.z, b1.z, c1.z, d1.z) B8(7, a1.w, b1.w, c1.w, d1.w)
#undef B8
}

// thread = one reference pixel x 8 channels; grid.z = depth chunks (gradients of the reference
// features are accumulated with atomics too, so chunks are independent).  h, w >= 2.
template <bool GWC>
__global__ void __launch_bounds__(128)
warp_cost_bwd_kernel(const float* __restrict__ feats,    // (B,V,h,w,C)
                     const float* __restrict__ proj,     // (B,V-1,3,4)
                     const float* __restrict__ dv,       // (B,D,h,w)
                     const float* __restrict__ gcost,    // (B,D,h,w,Cout)
                     float* __restrict__ gfeats,         // (B,V,h,w,C), accumulated into
                     int V, int C, int D, int h, int w, int G, int dchunk) {
  __shared__ float s_proj[15 * 12];
  const int b = blockIdx.y, nsrc = V - 1;
  for (int i = threadIdx.x; i < nsrc * 12; i += blockDim.x) s_proj[i] = proj[(size_t)b * nsrc * 12 + i];
  __syncthreads();
  const int tpp = C / 8;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int pix = gtid / tpp, c0 = (gtid - pix * tpp) * 8;
  const int hw = h * w;
  if (pix >= hw) return;
  const int y = pix / w, x = pix - y * w;
  const float xf = (float)x, yf = (float)y;
  const int row = w * C;
  const size_t vs = (size_t)hw * C;
  const float* fb = feats + (size_t)b * V * vs + c0;
  float* gb = gfeats + (size_t)b * V * vs + c0;
  float ref[8];
  {
    const float4 a = ldg4(fb + (size_t)pix * C), c = ldg4(fb + (size_t)pix * C + 4);
    ref[0] = a.x; ref[1] = a.y; ref[2] = a.z; ref[3] = a.w;
    ref[4] = c.x; ref[5] = c.y; ref[6] = c.z; ref[7] = c.w;
  }
  const float inv_v = 1.f / (float)V;
  const int cpg = GWC ? C / G : 1, cout = GWC ? G : C;
  const float gscale = GWC ? 1.f / ((float)cpg * (float)(V - 1)) : 0.f;
  float gref[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) gref[k] = 0.f;
  const int d0 = blockIdx.z * dchunk, d1 = min(D, d0 + dchunk);
  for (int d = d0; d < d1; ++d) {
    const float inv_d = rcp_approx(__ldg(dv + ((size_t)b * D + d) * hw + pix));
    // upstream gradient of this (pixel, plane) for the thread's 8 channels
    float g[8];
    const float* gp = gcost + ((size_t)(b * D + d) * hw + pix) * cout;
    if (!GWC) {
      const float4 a = ldg4(gp + c0), c = ldg4(gp + c0 + 4);
      g[0] = a.x; g[1] = a.y; g[2] = a.z; g[3] = a.w; g[4] = c.x; g[5] = c.y; g[6] = c.z; g[7] = c.w;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) g[k] = __ldg(gp + (c0 + k) / cpg) * gscale;
    }
    // pass 1: S = (ref +) sum of the warped views
    float S[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) S[k] = GWC ? 0.f : ref[k];
    for (int v = 0; v < nsrc; ++v) {
      const float* P = s_proj + v * 12;
      const float qx = fmaf(P[3], inv_d, fmaf(P[0], xf, fmaf(P[1], yf, P[2])));
      const float qy = fmaf(P[7], inv_d, fmaf(P[4], xf, fmaf(P[5], yf, P[6])));
      const float qz = fmaf(P[11], inv_d, fmaf(P[8], xf, fmaf(P[9], yf, P[10])));
      const TapPos t = tap_pos(qx, qy, qz, h, w, C);
      float r[8];
      blend8f(fb + (size_t)(v + 1) * vs + t.off, C, row, t, r);
#pragma unroll
      for (int k = 0; k < 8; ++k) S[k] += r[k];
    }
    if (!GWC) {
      // var = Q/V - (S/V)^2: d/d ref = 2 ref/V - 2 S/V^2 (ref is one of the summands)
#pragma unroll
      for (int k = 0; k < 8; ++k) gref[k] = fmaf(g[k], 2.f * inv_v * (ref[k] - S[k] * inv_v), gref[k]);
    } else {
      // cost_g = mean_c(S*ref)/(V-1): d/d ref = S * g/(cpg (V-1))
#pragma unroll
      for (int k = 0; k < 8; ++k) gref[k] = fmaf(g[k], S[k], gref[k]);
    }
    // pass 2: per view, d/d r_v scattered through the bilinear taps
    for (int v = 0; v < nsrc; ++v) {
      const float* P = s_proj + v * 12;
      const float qx = fmaf(P[3], inv_d, fmaf(P[0], xf, fmaf(P[1], yf, P[2])));
      const float qy = fmaf(P[7], inv_d, fmaf(P[4], xf, fmaf(P[5], yf, P[6])));
      const float qz = fmaf(P[11], inv_d, fmaf(P[8], xf, fmaf(P[9], yf, P[10])));
      const TapPos t = tap_pos(qx, qy, qz, h, w, C);
      if (t.w00 == 0.f && t.w01 == 0.f && t.w10 == 0.f && t.w11 == 0.f) continue;
      float coef[8];
      if (!GWC) {
        float r[8];
        blend8f(fb + (size_t)(v + 1) * vs + t.off, C, row, t, r);
#pragma unroll
        for (int k = 0; k < 8; ++k) coef[k] = g[k] * 2.f * inv_v * (r[k] - S[k] * inv_v);
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) coef[k] = g[k] * ref[k];
      }
      float* o = gb + (size_t)(v + 1) * vs + t.off;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        atomicAdd(o + k, coef[k] * t.w00);
        atomicAdd(o + C + k, coef[k] * t.w01);
        atomicAdd(o + row + k, coef[k] * t.w10);
        atomicAdd(o + row + C + k, coef[k] * t.w11);
      }
    }
  }
  float* o = gb + (size_t)pix * C;
#pragma unroll
  for (int k = 0; k < 8; ++k) atomicAdd(o + k, gref[k]);
}

// dW[tap][a][b] += sum over (batch, output voxel o) of X[s*o + k - 1][a] * G[o][b]
// X (B,Di,hi,wi,Ca), G (B,Do,ho,wo,Cb) channels-last; Ca, Cb <= 64.
// grid = (27 taps, voxel chunks); 256 threads = 16 (a, 4 each) x 16 (b, 4 each).
constexpr int kWgNV = 32;
__global__ void __launch_bounds__(256)
conv3d_wgrad_kernel(const float* __restrict__ X, const float* __restrict__ Gy,
                    float* __restrict__ dW, int B, int Ca, int Cb, int Di, int hi, int wi, int Do,
                    int ho, int wo, int stride, long chunk) {
  __shared__ float xs[kWgNV][64 + 1], gs[kWgNV][64 + 1];
  const int tap = blockIdx.x;
  const int kd = tap / 9, kh = (tap / 3) % 3, kw = tap % 3;
  const long total = (long)B * Do * ho * wo;
  const long v0 = (long)blockIdx.y * chunk, v1 = min(total, v0 + chunk);
  const int ta = threadIdx.x & 15, tb = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (long base = v0; base < v1; base += kWgNV) {
    __syncthreads();
    for (int i = threadIdx.x; i < kWgNV * 64; i += blockDim.x) {
      const int vv = i >> 6, c = i & 63;
      const long o = base + vv;
      float xv = 0.f, gv = 0.f;
      if (o < v1) {
        long t = o;
        const int ow = (int)(t % wo); t /= wo;
        const int oh = (int)(t % ho); t /= ho;
        const int od = (int)(t % Do);
        const int b = (int)(t / Do);
        const int id = stride * od + kd - 1, ih = stride * oh + kh - 1, iw = stride * ow + kw - 1;
        if (c < Cb) gv = __ldg(Gy + (size_t)o * Cb + c);
        if (c < Ca && id >= 0 && id < Di && ih >= 0 && ih < hi && iw >= 0 && iw < wi)
          xv = __ldg(X + ((((size_t)b * Di + id) * hi + ih) * wi + iw) * Ca + c);
      }
      xs[vv][c] = xv;
      gs[vv][c] = gv;
    }
    __syncthreads();
    if (ta * 4 < Ca && tb * 4 < Cb) {
#pragma unroll 4
      for (int vv = 0; vv < kWgNV; ++vv) {
        float a[4], g[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { a[i] = xs[vv][ta * 4 + i]; g[i] = gs[vv][tb * 4 + i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], g[j], acc[i][j]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int a = ta * 4 + i, bb = tb * 4 + j;
      if (a < Ca && bb < Cb) atomicAdd(dW + ((size_t)tap * Ca + a) * Cb + bb, acc[i][j]);
    }
}

// depth = sum_d softmax(l)_d * dv_d  =>  d depth / d l_d = p_d (dv_d - depth)
__global__ void __launch_bounds__(128)
regress_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ dv,
                   int dv_is_vector, const float* __restrict__ gdepth, float* __restrict__ glogits,
                   int D, int hw) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= hw) return;
  const float* lp = logits + (size_t)b * D * hw + pix;
  const float* dp = dv_is_vector ? dv : dv + (size_t)b * D * hw + pix;
  const size_t ds = dv_is_vector ? 1 : (size_t)hw;
  float m = -INFINITY;
  for (int d = 0; d < D; ++d) m = fmaxf(m, __ldg(lp + (size_t)d * hw));
  float den = 0.f, num = 0.f;
  for (int d = 0; d < D; ++d) {
    const float e = expf(__ldg(lp + (size_t)d * hw) - m);
    den += e;
    num = fmaf(e, __ldg(dp + d * ds), num);
  }
  const float depth = num / den, g = __ldg(gdepth + (size_t)b * hw + pix) / den;
  float* op = glogits + (size_t)b * D * hw + pix;
  for (int d = 0; d < D; ++d) {
    const float e = expf(__ldg(lp + (size_t)d * hw) - m);
    op[(size_t)d * hw] = e * (__ldg(dp + d * ds) - depth) * g;
  }
}

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_warp_cost_bwd(const float* feats, const float* proj, const float* depth_values,
                                    const float* grad_cost, float* grad_feats, int B, int V, int C,
                                    int D, int h, int w, int num_groups, void* stream) {
  CASMVS_REQUIRE(feats && proj && depth_values && grad_cost && grad_feats, "warp_cost_bwd: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && V >= 2 && V - 1 <= 15 && C > 0 && C % 8 == 0 && D > 0 &&
                     h >= 2 && w >= 2, "warp_cost_bwd: bad dims");
  CASMVS_REQUIRE(num_groups >= 1 && C % num_groups == 0, "warp_cost_bwd: C %% num_groups != 0");
  CASMVS_REQUIRE((size_t)h * w * C < (1u << 31), "warp_cost_bwd: view too large");
  if (B == 0) return 0;
  const long threads = (long)h * w * (C / 8);
  int dchunk = D;
  while (dchunk > 4 && (threads / 128 + 1) * B * ((D + dchunk - 1) / dchunk) < (long)num_sms() * 8)
    dchunk = (dchunk + 1) / 2;
  dim3 grd((unsigned)((threads + 127) / 128), (unsigned)B, (unsigned)((D + dchunk - 1) / dchunk));
  cudaStream_t st = as_stream(stream);
  if (num_groups > 1)
    warp_cost_bwd_kernel<true><<<grd, 128, 0, st>>>(feats, proj, depth_values, grad_cost, grad_feats,
                                                    V, C, D, h, w, num_groups, dchunk);
  else
    warp_cost_bwd_kernel<false><<<grd, 128, 0, st>>>(feats, proj, depth_values, grad_cost,
                                                     grad_feats, V, C, D, h, w, 1, dchunk);
  return after_launch("warp_cost_bwd");
}

extern "C" int casmvs_conv3d_wgrad(const float* x, const float* grad_y, float* grad_w, int B, int Ca,
                                   int Cb, int Di, int hi, int wi, int Do, int ho, int wo,
                                   int stride, void* stream) {
  CASMVS_REQUIRE(x && grad_y && grad_w, "conv3d_wgrad: null pointer");
  CASMVS_REQUIRE(B >= 0 && Ca > 0 && Ca <= 64 && Cb > 0 && Cb <= 64, "conv3d_wgrad: channels must be in 1..64");
  CASMVS_REQUIRE(stride == 1 || stride == 2, "conv3d_wgrad: stride must be 1 or 2");
  CASMVS_REQUIRE(Do == (Di - 1) / stride + 1 && ho == (hi - 1) / stride + 1 &&
                     wo == (wi - 1) / stride + 1, "conv3d_wgrad: output dims do not match");
  if (B == 0) return 0;
  const long total = (long)B * Do * ho * wo;
  long chunks = (long)num_sms() * 4 / 27 + 1;
  if (chunks > (total + kWgNV - 1) / kWgNV) chunks = (total + kWgNV - 1) / kWgNV;
  if (chunks < 1) chunks = 1;
  long chunk = (total + chunks - 1) / chunks;
  chunk = (chunk + kWgNV - 1) / kWgNV * kWgNV;
  chunks = (total + chunk - 1) / chunk;
  conv3d_wgrad_kernel<<<dim3(27, (unsigned)chunks), 256, 0, as_stream(stream)>>>(
      x, grad_y, grad_w, B, Ca, Cb, Di, hi, wi, Do, ho, wo, stride, chunk);
  return after_launch("conv3d_wgrad");
}

extern "C" int casmvs_regress_bwd(const float* logits, const float* depth_values, int dv_is_vector,
                                  const float* grad_depth, float* grad_logits, int B, int D, int h,
                                  int w, void* stream) {
  CASMVS_REQUIRE(logits && depth_values && grad_depth && grad_logits, "regress_bwd: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "regress_bwd: bad dims");
  if (B == 0) return 0;
  const int hw = h * w;
  regress_bwd_kernel<<<dim3((hw + 127) / 128, B), 128, 0, as_stream(stream)>>>(
      logits, depth_values, dv_is_vector, grad_depth, grad_logits, D, hw);
  return after_launch("regress_bwd");
}
