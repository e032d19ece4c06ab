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
//
// Deterministic variants (picked by autograd.py when torch's deterministic algorithms are on;
// DESIGN.md §3): the same bits for the same inputs and shapes, whatever the scheduling.
//   casmvs_warp_cost_bwd_det        contribution pass -> stable radix sort by destination
//                                   texel -> per-texel sum in contribution order
//   casmvs_conv3d_wgrad_det         per-chunk partials to a workspace, reduced in chunk order
//   casmvs_upsample2x_bilinear_bwd  FeatureNet's x2 upsample backward as a gather
#include <climits>

#include <cub/device/device_radix_sort.cuh>

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

// Where the K1 backward puts its two kinds of result: each (plane d, source view v) bilinear
// contribution coef[k] * w_tap for the 2x2 window t of view v, and the reference pixel's
// gradient summed over the thread's planes.  AtomicSink adds both into grad_feats; DetSink
// (casmvs_warp_cost_bwd_det) records the contributions for a fixed-order sum instead.
struct AtomicSink {
  float* gb;                     // grad_feats of batch item b, channel c0
  size_t vs;                     // floats per view
  int C, row;
  __device__ __forceinline__ void skip(int, int) const {}
  __device__ __forceinline__ void taps(int v, int, const TapPos& t, const float (&coef)[8]) const {
    float* o = gb + (size_t)(v + 1) * vs + t.off;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      atomicAdd(o + k, coef[k] * t.w00);
      atomicAdd(o + C + k, coef[k] * t.w01);
      atomicAdd(o + row + k, coef[k] * t.w10);
      atomicAdd(o + row + C + k, coef[k] * t.w11);
    }
  }
  __device__ __forceinline__ void ref(int pix, const float (&gref)[8]) const {
    float* o = gb + (size_t)pix * C;
#pragma unroll
    for (int k = 0; k < 8; ++k) atomicAdd(o + k, gref[k]);
  }
};

// Contribution ci = ((b*D + d)*hw + pix)*(V-1) + v has entries 4*ci + tap (taps nw, ne, sw, se).
// Entry e's key is its destination texel (b*(V-1) + v)*hw + texel, or `nkeys` when the sample
// has no weight (the atomic kernel skips it); wts[e] is the tap weight and coefs[ci*C + c] the
// coefficient.  Every slot is written by a fixed thread, so the arrays do not depend on timing.
struct DetSink {
  float* gb;                     // grad_feats of batch item b, channel c0 (reference view only)
  float* __restrict__ coefs;
  float* __restrict__ wts;
  unsigned* __restrict__ keys;
  unsigned* __restrict__ vals;
  size_t ci0;                    // contribution index of (b, d = 0, pix, v = 0)
  size_t dstride;                // contributions per plane: hw * (V-1)
  unsigned key0;                 // key of (b, v = 0, texel 0)
  unsigned nkeys;
  int C, c0, w, hw;
  __device__ __forceinline__ size_t index(int v, int d) const { return ci0 + d * dstride + v; }
  __device__ __forceinline__ void skip(int v, int d) const {
    if (c0) return;
    const size_t e = 4 * index(v, d);
#pragma unroll
    for (int k = 0; k < 4; ++k) { keys[e + k] = nkeys; vals[e + k] = (unsigned)(e + k); }
  }
  __device__ __forceinline__ void taps(int v, int d, const TapPos& t, const float (&coef)[8]) const {
    const size_t ci = index(v, d);
    float4* cp = reinterpret_cast<float4*>(coefs + ci * C + c0);
    cp[0] = make_float4(coef[0], coef[1], coef[2], coef[3]);
    cp[1] = make_float4(coef[4], coef[5], coef[6], coef[7]);
    if (c0) return;
    const unsigned k0 = key0 + (unsigned)v * hw + t.off / C;
    const size_t e = 4 * ci;
    keys[e] = k0; keys[e + 1] = k0 + 1; keys[e + 2] = k0 + w; keys[e + 3] = k0 + w + 1;
    *reinterpret_cast<float4*>(wts + e) = make_float4(t.w00, t.w01, t.w10, t.w11);
#pragma unroll
    for (int k = 0; k < 4; ++k) vals[e + k] = (unsigned)(e + k);
  }
  __device__ __forceinline__ void ref(int pix, const float (&gref)[8]) const {
    float4* o = reinterpret_cast<float4*>(gb + (size_t)pix * C);
    o[0] = make_float4(gref[0], gref[1], gref[2], gref[3]);
    o[1] = make_float4(gref[4], gref[5], gref[6], gref[7]);
  }
};

// One reference pixel x 8 channels over planes [d0, d1): pass 1 forms the sum S of the warped
// views, pass 2 hands each view's bilinear contribution to the sink.  h, w >= 2.
template <bool GWC, class Sink>
__device__ __forceinline__ void
warp_cost_bwd_pixel(const float* __restrict__ s_proj, const float* __restrict__ fb,
                    const float* __restrict__ dv, const float* __restrict__ gcost, int b, int pix,
                    int c0, int V, int C, int D, int h, int w, int G, int d0, int d1,
                    const Sink& sink) {
  const int nsrc = V - 1;
  const int hw = h * w;
  const int y = pix / w, x = pix - y * w;
  const float xf = (float)x, yf = (float)y;
  const int row = w * C;
  const size_t vs = (size_t)hw * C;
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
      if (t.w00 == 0.f && t.w01 == 0.f && t.w10 == 0.f && t.w11 == 0.f) {
        sink.skip(v, d);
        continue;
      }
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
      sink.taps(v, d, t, coef);
    }
  }
  sink.ref(pix, gref);
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
  const size_t vs = (size_t)hw * C;
  const AtomicSink sink{gfeats + (size_t)b * V * vs + c0, vs, C, w * C};
  const int d0 = blockIdx.z * dchunk, d1 = min(D, d0 + dchunk);
  warp_cost_bwd_pixel<GWC>(s_proj, feats + (size_t)b * V * vs + c0, dv, gcost, b, pix, c0, V, C, D,
                           h, w, G, d0, d1, sink);
}

// Contribution pass of casmvs_warp_cost_bwd_det: the same threads as warp_cost_bwd_kernel, each
// walking all D planes, so the reference-view gradient is summed in plane order and stored.
template <bool GWC>
__global__ void __launch_bounds__(128)
warp_cost_bwd_det_kernel(const float* __restrict__ feats, const float* __restrict__ proj,
                         const float* __restrict__ dv, const float* __restrict__ gcost,
                         float* __restrict__ gfeats, float* __restrict__ coefs,
                         float* __restrict__ wts, unsigned* __restrict__ keys,
                         unsigned* __restrict__ vals, int V, int C, int D, int h, int w, int G) {
  __shared__ float s_proj[15 * 12];
  const int b = blockIdx.y, nsrc = V - 1;
  for (int i = threadIdx.x; i < nsrc * 12; i += blockDim.x) s_proj[i] = proj[(size_t)b * nsrc * 12 + i];
  __syncthreads();
  const int tpp = C / 8;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int pix = gtid / tpp, c0 = (gtid - pix * tpp) * 8;
  const int hw = h * w;
  if (pix >= hw) return;
  const size_t vs = (size_t)hw * C;
  const DetSink sink{gfeats + (size_t)b * V * vs + c0, coefs, wts, keys, vals,
                     ((size_t)b * D * hw + pix) * nsrc, (size_t)hw * nsrc,
                     (unsigned)(b * nsrc * hw), (unsigned)(gridDim.y * nsrc * hw), C, c0, w, hw};
  warp_cost_bwd_pixel<GWC>(s_proj, feats + (size_t)b * V * vs + c0, dv, gcost, b, pix, c0, V, C, D,
                           h, w, G, 0, D, sink);
}

// sorted keys -> [begin, end) of every destination texel's run (texels without contributions
// keep the zeroed empty range)
__global__ void seg_bounds_kernel(const unsigned* __restrict__ keys, unsigned n, unsigned nkeys,
                                  unsigned* __restrict__ begin, unsigned* __restrict__ end) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned k = keys[i];
  if (k >= nkeys) return;
  if (i == 0 || keys[i - 1] != k) begin[k] = i;
  if (i + 1 == n || keys[i + 1] != k) end[k] = i + 1;
}

// thread = one source-view texel x 8 channels: the run's contributions coef * w_tap added one
// by one in entry order (a stable sort keeps the contribution-index order inside a run), each
// product rounded before the add as the atomic kernel's are.
__global__ void __launch_bounds__(128)
warp_cost_bwd_gather_kernel(const unsigned* __restrict__ vals, const unsigned* __restrict__ begin,
                            const unsigned* __restrict__ end, const float* __restrict__ coefs,
                            const float* __restrict__ wts, float* __restrict__ gfeats, int V,
                            int C, int hw, long nthreads) {
  const long gtid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gtid >= nthreads) return;
  const int tpp = C / 8, nsrc = V - 1;
  const long key = gtid / tpp;
  const int c0 = (int)(gtid - key * tpp) * 8;
  const int texel = (int)(key % hw);
  const long bv = key / hw;
  const int b = (int)(bv / nsrc), v = (int)(bv - (long)b * nsrc);
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  const unsigned e1 = end[key];
  for (unsigned e = begin[key]; e < e1; ++e) {
    const unsigned u = vals[e];
    const float wt = __ldg(wts + u);
    const float4* cp = reinterpret_cast<const float4*>(coefs + (size_t)(u >> 2) * C + c0);
    const float4 a = __ldg(cp), c = __ldg(cp + 1);
    const float cf[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = __fadd_rn(acc[k], __fmul_rn(cf[k], wt));
  }
  float4* o = reinterpret_cast<float4*>(gfeats + (((size_t)b * V + v + 1) * hw + texel) * C + c0);
  o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// dW[tap][a][b] += sum over (batch, output voxel o) of X[s*o + k - 1][a] * G[o][b]
// X (B,Di,hi,wi,Ca), G (B,Do,ho,wo,Cb) channels-last; Ca, Cb <= 64.
// grid = (27 taps, voxel chunks); 256 threads = 16 (a, 4 each) x 16 (b, 4 each).
// part == NULL: each chunk's sums are added into dW with atomics.  Otherwise chunk c stores its
// sums to part[c][tap][a][b] and wgrad_reduce_kernel adds the chunks up in order.
constexpr int kWgNV = 32;
__global__ void __launch_bounds__(256)
conv3d_wgrad_kernel(const float* __restrict__ X, const float* __restrict__ Gy,
                    float* __restrict__ dW, float* __restrict__ part, int B, int Ca, int Cb, int Di,
                    int hi, int wi, int Do, int ho, int wo, int stride, long chunk) {
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
      // each tile of kWgNV voxels is summed on its own, then added to the running sum: a CTA
      // sums ~10^5 voxels per tap at training sizes, and one sequential fp32 sum over all of
      // them loses ~sqrt(n) ulps of sum |x| |gy| when the terms share a sign (kernel input and
      // gradient both non-negative), ~sqrt(n / kWgNV) this way
      float part[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) part[i][j] = 0.f;
#pragma unroll 4
      for (int vv = 0; vv < kWgNV; ++vv) {
        float a[4], g[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { a[i] = xs[vv][ta * 4 + i]; g[i] = gs[vv][tb * 4 + i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) part[i][j] = fmaf(a[i], g[j], part[i][j]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += part[i][j];
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int a = ta * 4 + i, bb = tb * 4 + j;
      if (a >= Ca || bb >= Cb) continue;
      const size_t o = ((size_t)tap * Ca + a) * Cb + bb;
      if (part)
        part[(size_t)blockIdx.y * gridDim.x * Ca * Cb + o] = acc[i][j];
      else
        atomicAdd(dW + o, acc[i][j]);
    }
}

// dW[i] = sum over chunks c = 0, 1, ... of part[c][i], in that order
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dW, int n,
                                    int chunks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += __ldg(part + (size_t)c * n + i);
  dW[i] = s;
}

// Voxel chunks of the deterministic weight gradient, from the voxel count alone: chunks of
// kWgDetTiles tiles, at most kWgDetMaxChunks of them (longer chunks beyond that).
constexpr long kWgDetTiles = 64, kWgDetMaxChunks = 2048;
inline void wgrad_det_chunks(long total, long* chunk, long* chunks) {
  const long tiles = (total + kWgNV - 1) / kWgNV;
  long n = (tiles + kWgDetTiles - 1) / kWgDetTiles;
  if (n > kWgDetMaxChunks) n = kWgDetMaxChunks;
  if (n < 1) n = 1;
  const long per = (tiles + n - 1) / n;
  *chunk = per * kWgNV;
  *chunks = per ? (tiles + per - 1) / per : 1;
}

// grad_x of y = upsample_bilinear2d(x, 2h x 2w, align_corners=True) as a gather: thread = one
// input element, which adds the contributions of the output pixels that read it (rows 2y-3 ..
// 2y+4 and the same columns cover them) in output order, each tap's weight and product formed
// as ATen's forward and backward form them, taps in ATen's order (h1,w1), (h1,w1+w1p),
// (h1+h1p,w1), (h1+h1p,w1+w1p).  nhwc: both tensors channels-last, else NCHW.
__global__ void upsample2x_bilinear_bwd_kernel(const float* __restrict__ gy, float* __restrict__ gx,
                                               int N, int C, int h, int w, float sh, float sw,
                                               int nhwc) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)N * C * h * w) return;
  int n, c, y, x;
  long t = i;
  if (nhwc) {
    c = (int)(t % C); t /= C; x = (int)(t % w); t /= w; y = (int)(t % h); n = (int)(t / h);
  } else {
    x = (int)(t % w); t /= w; y = (int)(t % h); t /= h; c = (int)(t % C); n = (int)(t / C);
  }
  const int H = 2 * h, W = 2 * w;
  auto at = [&](int oy, int ox) {
    return nhwc ? gy[(((size_t)n * H + oy) * W + ox) * C + c]
                : gy[(((size_t)n * C + c) * H + oy) * W + ox];
  };
  float acc = 0.f;
  for (int oy = max(0, 2 * y - 3); oy <= min(H - 1, 2 * y + 4); ++oy) {
    const float h1r = sh * oy;
    const int h1 = (int)h1r;
    const int h1p = (h1 < h - 1) ? 1 : 0;
    const float l1h = h1r - h1, l0h = 1.f - l1h;
    const bool top = h1 == y, bottom = h1 + h1p == y;
    if (!top && !bottom) continue;
    for (int ox = max(0, 2 * x - 3); ox <= min(W - 1, 2 * x + 4); ++ox) {
      const float w1r = sw * ox;
      const int w1 = (int)w1r;
      const int w1p = (w1 < w - 1) ? 1 : 0;
      const float l1w = w1r - w1, l0w = 1.f - l1w;
      const bool left = w1 == x, right = w1 + w1p == x;
      if (!left && !right) continue;
      const float g = at(oy, ox);
      if (top && left) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(l0h, l0w), g));
      if (top && right) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(l0h, l1w), g));
      if (bottom && left) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(l1h, l0w), g));
      if (bottom && right) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(l1h, l1w), g));
    }
  }
  gx[i] = acc;
}

// inverse depth (regress.cu, rule 5): ubar = sum_d p_d RN(1/dv_d), depth = RN(1/ubar)
//   =>  d depth / d l_d = -depth^2 p_d (RN(1/dv_d) - ubar)
__global__ void __launch_bounds__(128)
regress_inv_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ dv,
                       int dv_is_vector, const float* __restrict__ gdepth,
                       float* __restrict__ glogits, int D, int hw) {
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
    num = fmaf(e, __frcp_rn(__ldg(dp + d * ds)), num);
  }
  const float ubar = num / den, depth = __frcp_rn(ubar);
  const float g = -(depth * depth) * (__ldg(gdepth + (size_t)b * hw + pix) / den);
  float* op = glogits + (size_t)b * D * hw + pix;
  for (int d = 0; d < D; ++d) {
    const float e = expf(__ldg(lp + (size_t)d * hw) - m);
    op[(size_t)d * hw] = e * (__frcp_rn(__ldg(dp + d * ds)) - ubar) * g;
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
      x, grad_y, grad_w, nullptr, B, Ca, Cb, Di, hi, wi, Do, ho, wo, stride, chunk);
  return after_launch("conv3d_wgrad");
}

extern "C" size_t casmvs_conv3d_wgrad_det_workspace_bytes(int B, int Ca, int Cb, int Do, int ho,
                                                         int wo) {
  if (B <= 0 || Ca <= 0 || Cb <= 0 || Do <= 0 || ho <= 0 || wo <= 0) return 0;
  long chunk, chunks;
  wgrad_det_chunks((long)B * Do * ho * wo, &chunk, &chunks);
  return (size_t)chunks * 27 * Ca * Cb * sizeof(float);
}

extern "C" int casmvs_conv3d_wgrad_det(const float* x, const float* grad_y, float* grad_w, int B,
                                       int Ca, int Cb, int Di, int hi, int wi, int Do, int ho,
                                       int wo, int stride, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  CASMVS_REQUIRE(x && grad_y && grad_w, "conv3d_wgrad_det: null pointer");
  CASMVS_REQUIRE(B >= 0 && Ca > 0 && Ca <= 64 && Cb > 0 && Cb <= 64, "conv3d_wgrad_det: channels must be in 1..64");
  CASMVS_REQUIRE(stride == 1 || stride == 2, "conv3d_wgrad_det: stride must be 1 or 2");
  CASMVS_REQUIRE(Do == (Di - 1) / stride + 1 && ho == (hi - 1) / stride + 1 &&
                     wo == (wi - 1) / stride + 1, "conv3d_wgrad_det: output dims do not match");
  const int n = 27 * Ca * Cb;
  cudaStream_t st = as_stream(stream);
  if (B == 0) {
    if (cudaMemsetAsync(grad_w, 0, (size_t)n * sizeof(float), st) != cudaSuccess)
      return after_launch("conv3d_wgrad_det");
    return 0;
  }
  CASMVS_REQUIRE(workspace && workspace_bytes >= casmvs_conv3d_wgrad_det_workspace_bytes(B, Ca, Cb, Do, ho, wo),
                 "conv3d_wgrad_det: workspace smaller than casmvs_conv3d_wgrad_det_workspace_bytes");
  long chunk, chunks;
  wgrad_det_chunks((long)B * Do * ho * wo, &chunk, &chunks);
  float* part = static_cast<float*>(workspace);
  conv3d_wgrad_kernel<<<dim3(27, (unsigned)chunks), 256, 0, st>>>(
      x, grad_y, grad_w, part, B, Ca, Cb, Di, hi, wi, Do, ho, wo, stride, chunk);
  if (int rc = after_launch("conv3d_wgrad_det")) return rc;
  wgrad_reduce_kernel<<<(n + 255) / 256, 256, 0, st>>>(part, grad_w, n, (int)chunks);
  return after_launch("conv3d_wgrad_det reduce");
}

namespace {
// Workspace of casmvs_warp_cost_bwd_det, in this order, each part 256-byte aligned: coefs
// (contributions x C floats), wts, keys, sorted keys, vals, sorted vals (4 per contribution),
// run begin / end per destination texel, then the radix sort's temporary storage.
struct BwdDetLayout {
  size_t n_contrib, n_ent, nkeys, off[9];
  int end_bit;
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

bool bwd_det_layout(int B, int V, int C, int D, int h, int w, BwdDetLayout* L) {
  const size_t hw = (size_t)h * w, nsrc = (size_t)(V - 1);
  L->n_contrib = (size_t)B * D * hw * nsrc;
  L->n_ent = 4 * L->n_contrib;
  L->nkeys = (size_t)B * nsrc * hw;
  if (L->n_ent > (size_t)INT_MAX || L->nkeys >= (size_t)UINT_MAX) return false;
  L->end_bit = 1;
  while (L->end_bit < 32 && (L->nkeys >> L->end_bit) != 0) ++L->end_bit;
  const size_t sizes[8] = {L->n_contrib * C * 4, L->n_ent * 4, L->n_ent * 4, L->n_ent * 4,
                           L->n_ent * 4, L->n_ent * 4, L->nkeys * 4, L->nkeys * 4};
  L->off[0] = 0;
  for (int i = 0; i < 8; ++i) L->off[i + 1] = L->off[i] + align256(sizes[i]);
  return true;
}

size_t sort_temp_bytes(const BwdDetLayout& L) {
  size_t bytes = 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const unsigned*)nullptr, (unsigned*)nullptr,
                                      (const unsigned*)nullptr, (unsigned*)nullptr,
                                      (int)L.n_ent, 0, L.end_bit) != cudaSuccess)
    return 0;
  return bytes;
}
}  // namespace

extern "C" size_t casmvs_warp_cost_bwd_det_workspace_bytes(int B, int V, int C, int D, int h, int w) {
  BwdDetLayout L;
  if (B <= 0 || V < 2 || C <= 0 || D <= 0 || h <= 0 || w <= 0) return 0;
  if (!bwd_det_layout(B, V, C, D, h, w, &L)) return 0;
  const size_t tmp = sort_temp_bytes(L);
  return tmp ? L.off[8] + tmp : 0;
}

extern "C" int casmvs_warp_cost_bwd_det(const float* feats, const float* proj,
                                        const float* depth_values, const float* grad_cost,
                                        float* grad_feats, int B, int V, int C, int D, int h, int w,
                                        int num_groups, void* workspace, size_t workspace_bytes,
                                        void* stream) {
  CASMVS_REQUIRE_ALIGNED("warp_cost_bwd_det", feats, 16);
  CASMVS_REQUIRE_ALIGNED("warp_cost_bwd_det", grad_feats, 16);
  CASMVS_REQUIRE_ALIGNED("warp_cost_bwd_det", workspace, 256);
  CASMVS_REQUIRE(feats && proj && depth_values && grad_cost && grad_feats, "warp_cost_bwd_det: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && V >= 2 && V - 1 <= 15 && C > 0 && C % 8 == 0 && D > 0 &&
                     h >= 2 && w >= 2, "warp_cost_bwd_det: bad dims");
  CASMVS_REQUIRE(num_groups >= 1 && C % num_groups == 0, "warp_cost_bwd_det: C %% num_groups != 0");
  CASMVS_REQUIRE((size_t)h * w * C < (1u << 31), "warp_cost_bwd_det: view too large");
  if (B == 0) return 0;
  BwdDetLayout L;
  CASMVS_REQUIRE(bwd_det_layout(B, V, C, D, h, w, &L), "warp_cost_bwd_det: too many contributions");
  const size_t need = casmvs_warp_cost_bwd_det_workspace_bytes(B, V, C, D, h, w);
  CASMVS_REQUIRE(need && workspace && workspace_bytes >= need,
                 "warp_cost_bwd_det: workspace smaller than casmvs_warp_cost_bwd_det_workspace_bytes");
  char* ws = static_cast<char*>(workspace);
  float* coefs = reinterpret_cast<float*>(ws + L.off[0]);
  float* wts = reinterpret_cast<float*>(ws + L.off[1]);
  unsigned* keys = reinterpret_cast<unsigned*>(ws + L.off[2]);
  unsigned* keys_sorted = reinterpret_cast<unsigned*>(ws + L.off[3]);
  unsigned* vals = reinterpret_cast<unsigned*>(ws + L.off[4]);
  unsigned* vals_sorted = reinterpret_cast<unsigned*>(ws + L.off[5]);
  unsigned* begin = reinterpret_cast<unsigned*>(ws + L.off[6]);
  unsigned* end = reinterpret_cast<unsigned*>(ws + L.off[7]);
  cudaStream_t st = as_stream(stream);

  const long threads = (long)h * w * (C / 8);
  dim3 grd((unsigned)((threads + 127) / 128), (unsigned)B, 1);
  if (num_groups > 1)
    warp_cost_bwd_det_kernel<true><<<grd, 128, 0, st>>>(feats, proj, depth_values, grad_cost,
                                                        grad_feats, coefs, wts, keys, vals, V, C,
                                                        D, h, w, num_groups);
  else
    warp_cost_bwd_det_kernel<false><<<grd, 128, 0, st>>>(feats, proj, depth_values, grad_cost,
                                                         grad_feats, coefs, wts, keys, vals, V, C,
                                                         D, h, w, 1);
  if (int rc = after_launch("warp_cost_bwd_det")) return rc;
  size_t tmp_bytes = workspace_bytes - L.off[8];
  cudaError_t e = cub::DeviceRadixSort::SortPairs(ws + L.off[8], tmp_bytes, keys, keys_sorted, vals,
                                                  vals_sorted, (int)L.n_ent, 0, L.end_bit, st);
  if (e != cudaSuccess) {
    set_error("warp_cost_bwd_det: radix sort failed: %s", cudaGetErrorString(e));
    return -2;
  }
  if (int rc = after_launch("warp_cost_bwd_det sort")) return rc;
  if (cudaMemsetAsync(begin, 0, L.off[8] - L.off[6], st) != cudaSuccess)
    return after_launch("warp_cost_bwd_det memset");
  seg_bounds_kernel<<<(unsigned)((L.n_ent + 255) / 256), 256, 0, st>>>(
      keys_sorted, (unsigned)L.n_ent, (unsigned)L.nkeys, begin, end);
  if (int rc = after_launch("warp_cost_bwd_det bounds")) return rc;
  const long gthreads = (long)L.nkeys * (C / 8);
  warp_cost_bwd_gather_kernel<<<(unsigned)((gthreads + 127) / 128), 128, 0, st>>>(
      vals_sorted, begin, end, coefs, wts, grad_feats, V, C, h * w, gthreads);
  return after_launch("warp_cost_bwd_det gather");
}

extern "C" int casmvs_upsample2x_bilinear_bwd(const float* grad_y, float* grad_x, int N, int C,
                                              int h, int w, int layout, void* stream) {
  CASMVS_REQUIRE(grad_y && grad_x, "upsample2x_bilinear_bwd: null pointer");
  CASMVS_REQUIRE(N >= 0 && C > 0 && h > 0 && w > 0, "upsample2x_bilinear_bwd: bad dims");
  CASMVS_REQUIRE(layout == CASMVS_NCHW || layout == CASMVS_NHWC, "upsample2x_bilinear_bwd: bad layout");
  const long n = (long)N * C * h * w;
  if (n == 0) return 0;
  // ATen's align_corners scale, (in - 1) / (out - 1) in float, computed on the host as there
  const float sh = (float)(h - 1) / (2 * h - 1), sw = (float)(w - 1) / (2 * w - 1);
  upsample2x_bilinear_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(
      grad_y, grad_x, N, C, h, w, sh, sw, layout == CASMVS_NHWC);
  return after_launch("upsample2x_bilinear_bwd");
}

extern "C" int casmvs_regress_bwd(const float* logits, const float* depth_values, int dv_is_vector,
                                  const float* grad_depth, float* grad_logits, int B, int D, int h,
                                  int w, void* stream) {
  CASMVS_REQUIRE(logits && depth_values && grad_depth && grad_logits, "regress_bwd: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0, "regress_bwd: bad dims");
  CASMVS_REQUIRE((dv_is_vector & ~(1 | CASMVS_INVERSE_DEPTH)) == 0, "regress_bwd: bad dv_is_vector flags");
  if (B == 0) return 0;
  const int hw = h * w;
  if (dv_is_vector & CASMVS_INVERSE_DEPTH) {
    regress_inv_bwd_kernel<<<dim3((hw + 127) / 128, B), 128, 0, as_stream(stream)>>>(
        logits, depth_values, dv_is_vector & 1, grad_depth, grad_logits, D, hw);
    return after_launch("regress_bwd");
  }
  regress_bwd_kernel<<<dim3((hw + 127) / 128, B), 128, 0, as_stream(stream)>>>(
      logits, depth_values, dv_is_vector, grad_depth, grad_logits, D, hw);
  return after_launch("regress_bwd");
}
