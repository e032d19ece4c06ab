// Self-supervised photometric loss (Khot et al. 2019; SSIM + L1 as Monodepth2) with a top-K
// over the source views and an edge-aware depth smoothness term.  The rule:
//
//   Level l < levels has h_l x w_l = H/2^l x W/2^l; level-l pixel (x, y) is level-0 pixel
//   (2^l x, 2^l y) of the network input (a strided subsample: the K of io.pyramid_proj_mats).
//   I = x * std_c + mean_c un-normalises the input with the ImageNet statistics.
//   Warp (homo_warp): p = R (x, y, 1) + T / d, u = p_x / p_z, v = p_y / p_z with (R | T) =
//   proj[b, s, l]; valid when d is finite and > 0, p_z > 1e-7, 0 <= u <= w_l - 1 and
//   0 <= v <= h_l - 1.  Bilinear with x0 = floor(u), tap x0 + 1 clamped to w_l - 1 (weight 0
//   there), the same in y; the derivative uses the same taps.
//   (q, s) is valid when q is off the 1-pixel border and all 9 samples of its 3x3 window N(q)
//   are valid (and its e below is finite, which only non-finite input breaks).  Per channel,
//   x = reference, y = warped source over N(q); mu and the centred (population, /9) variances
//   and covariance over N(q);
//     SSIM_c = (2 mu_x mu_y + C1)(2 s_xy + C2) / ((mu_x^2 + mu_y^2 + C1)(s_x^2 + s_y^2 + C2)),
//     C1 = 0.01^2, C2 = 0.03^2,
//     e_{q,s} = 0.85 mean_c (1 - SSIM_c) / 2 + 0.15 mean_c |x_c(q) - y_c(q)|.
//   Top-K: the valid sources ordered by (e, source index), the first min(K, n_valid) selected;
//   loss_q is their mean.  N_l counts the (b, q) with n_valid >= 1; P_l = sum loss_q / N_l
//   (0 when N_l = 0).
//   Smoothness on d^ = depth_l / (depth_interval[b] * interval_ratios[l]):
//     S_l = sum |d^(x+1,y) - d^(x,y)| exp(-g_x) / (B h_l (w_l - 1)) + the same in y over
//     (B (h_l - 1) w_l), g_x = mean_c |I_ref,c(x+1, y) - I_ref,c(x, y)|.
//   L = sum_l 2^(1-l) (P_l + lambda S_l); d|t|/dt at 0 is 0; only depth_l gets a gradient.
//
// Forward: one block per 16x16 tile of one (b, level).  The reference tile and, per source, the
// warped tile are staged in shared memory with a 1-pixel halo; each thread keeps its pixel's
// running top-K in registers.  Per-block sums are fp64 reduced in a fixed order, then one block
// finishes the levels (as loss.cu does), so the outputs are the same bits run to run.  The
// forward saves the per-pixel selection (uint16, bit s = source s) and N_l on the device.
// Backward: a pure gather per pixel p.  Per source, the warped tile is staged with a 2-pixel
// halo, the SSIM coefficients of every window q with s selected are recomputed once per q, and
// p sums the terms of the 9 windows containing it.  No atomics anywhere.
#include <cstdint>

#include "common.cuh"

namespace casmvs {

constexpr int kPhotoTile = 16;
constexpr int kPhotoThreads = kPhotoTile * kPhotoTile;
constexpr int kPhotoMaxLevels = 4;
constexpr int kPhotoMaxSources = 16;
constexpr int kPhotoSlots = 4;        // per block: sum loss_q, #valid pixels, smooth x, smooth y
constexpr float kPhotoAlpha = 0.85f;
constexpr float kPhotoC1 = 0.01f * 0.01f;
constexpr float kPhotoC2 = 0.03f * 0.03f;
__constant__ float kPhotoMean[3] = {0.485f, 0.456f, 0.406f};   // io.IMAGENET_MEAN / _STD
__constant__ float kPhotoStd[3] = {0.229f, 0.224f, 0.225f};

struct PhotoLevels {
  const float* depth[kPhotoMaxLevels];
  float* grad[kPhotoMaxLevels];
  uint16_t* sel[kPhotoMaxLevels];
  float* dbg_e[kPhotoMaxLevels];          // (B,S,h,w), NaN where (q, s) is not valid
  uint16_t* dbg_valid[kPhotoMaxLevels];   // (B,h,w), bit s = (q, s) valid
  float* dbg_lossq[kPhotoMaxLevels];      // (B,h,w), NaN where no source is valid
  float ratio[kPhotoMaxLevels];
  int h[kPhotoMaxLevels], w[kPhotoMaxLevels], tiles_x[kPhotoMaxLevels], tiles_y[kPhotoMaxLevels];
  int begin[kPhotoMaxLevels + 1];         // first block of each level
  int levels;
};

struct PhotoArgs {
  const float* imgs;     // (B,V,3,H,W) normalised
  const float* proj;     // (B,S,levels,3,4)
  const float* dint;     // (B)
  int B, S, H, W, K;
  float lambda;
};

struct Tile {
  int l, b, x0, y0, h, w;
};

__device__ __forceinline__ Tile tile_of(const PhotoLevels& L) {
  Tile t;
  const int blk = blockIdx.x;
  int l = 0;
  while (l + 1 < L.levels && blk >= L.begin[l + 1]) ++l;
  const int local = blk - L.begin[l];
  t.l = l;
  t.h = L.h[l];
  t.w = L.w[l];
  t.x0 = (local % L.tiles_x[l]) * kPhotoTile;
  const int rest = local / L.tiles_x[l];
  t.y0 = (rest % L.tiles_y[l]) * kPhotoTile;
  t.b = rest / L.tiles_y[l];
  return t;
}

// Un-normalised channel c of view v at level-l pixel (x, y).
__device__ __forceinline__ float image_at(const PhotoArgs& A, int b, int v, int c, int l, int x, int y) {
  const size_t V = (size_t)A.S + 1;
  const float n = __ldg(A.imgs + (((b * V + v) * 3 + c) * A.H + ((size_t)y << l)) * A.W + ((size_t)x << l));
  return __fadd_rn(__fmul_rn(n, kPhotoStd[c]), kPhotoMean[c]);
}

struct WarpPt {
  bool ok;
  int x0, y0, x1, y1;
  float fx, fy, u, v, pz, inv_d;
};

__device__ __forceinline__ WarpPt warp_point(const float* P, int x, int y, float d, int w, int h) {
  WarpPt r;
  r.ok = false;
  if (!(isfinite(d) && d > 0.f)) return r;
  r.inv_d = __frcp_rn(d);
  const float xf = (float)x, yf = (float)y;
  const float px = fmaf(P[3], r.inv_d, fmaf(P[0], xf, fmaf(P[1], yf, P[2])));
  const float py = fmaf(P[7], r.inv_d, fmaf(P[4], xf, fmaf(P[5], yf, P[6])));
  const float pz = fmaf(P[11], r.inv_d, fmaf(P[8], xf, fmaf(P[9], yf, P[10])));
  if (!(pz > 1e-7f)) return r;
  const float u = __fdiv_rn(px, pz), v = __fdiv_rn(py, pz);
  if (!(u >= 0.f && u <= (float)(w - 1) && v >= 0.f && v <= (float)(h - 1))) return r;
  r.ok = true;
  r.u = u;
  r.v = v;
  r.pz = pz;
  const float fu = floorf(u), fv = floorf(v);
  r.x0 = (int)fu;
  r.y0 = (int)fv;
  r.fx = u - fu;
  r.fy = v - fv;
  r.x1 = min(r.x0 + 1, w - 1);
  r.y1 = min(r.y0 + 1, h - 1);
  return r;
}

struct Taps4 {
  float v00, v01, v10, v11;
};

__device__ __forceinline__ Taps4 taps(const PhotoArgs& A, int b, int s, int c, int l, const WarpPt& p) {
  return {image_at(A, b, s + 1, c, l, p.x0, p.y0), image_at(A, b, s + 1, c, l, p.x1, p.y0),
          image_at(A, b, s + 1, c, l, p.x0, p.y1), image_at(A, b, s + 1, c, l, p.x1, p.y1)};
}

__device__ __forceinline__ float bilinear(const Taps4& t, const WarpPt& p) {
  const float top = fmaf(p.fx, t.v01 - t.v00, t.v00);
  const float bot = fmaf(p.fx, t.v11 - t.v10, t.v10);
  return fmaf(p.fy, bot - top, top);
}

struct WinStats {
  float mx, my, sxx, syy, sxy;
};

// Window statistics of channel c over the 3x3 window centred at (cx, cy) of two staged tiles.
template <int N>
__device__ __forceinline__ WinStats window_stats(const float (*x)[N][N], const float (*y)[N][N], int c,
                                                 int cx, int cy) {
  float mx = 0.f, my = 0.f;
#pragma unroll
  for (int j = -1; j <= 1; ++j)
#pragma unroll
    for (int i = -1; i <= 1; ++i) {
      mx += x[c][cy + j][cx + i];
      my += y[c][cy + j][cx + i];
    }
  mx *= (1.f / 9.f);
  my *= (1.f / 9.f);
  float sxx = 0.f, syy = 0.f, sxy = 0.f;
#pragma unroll
  for (int j = -1; j <= 1; ++j)
#pragma unroll
    for (int i = -1; i <= 1; ++i) {
      const float a = x[c][cy + j][cx + i] - mx, b = y[c][cy + j][cx + i] - my;
      sxx = fmaf(a, a, sxx);
      syy = fmaf(b, b, syy);
      sxy = fmaf(a, b, sxy);
    }
  return {mx, my, sxx * (1.f / 9.f), syy * (1.f / 9.f), sxy * (1.f / 9.f)};
}

__device__ __forceinline__ float depth_hat(float d, float delta) { return __fdiv_rn(d, delta); }

__device__ __forceinline__ float sgnf(float t) { return t > 0.f ? 1.f : (t < 0.f ? -1.f : 0.f); }

// Fixed-order block sum of kPhotoSlots doubles per thread; result in red[slot * kPhotoThreads].
__device__ void photo_block_reduce(double (&v)[kPhotoSlots], double* red) {
  const int t = threadIdx.x;
#pragma unroll
  for (int s = 0; s < kPhotoSlots; ++s) red[s * kPhotoThreads + t] = v[s];
  __syncthreads();
  for (int half = kPhotoThreads / 2; half > 0; half >>= 1) {
    if (t < half) {
#pragma unroll
      for (int s = 0; s < kPhotoSlots; ++s) red[s * kPhotoThreads + t] += red[s * kPhotoThreads + t + half];
    }
    __syncthreads();
  }
}

constexpr int kF = kPhotoTile + 2;   // forward tile with a 1-pixel halo
constexpr int kG = kPhotoTile + 4;   // backward tile with a 2-pixel halo

__global__ void __launch_bounds__(kPhotoThreads) photo_fwd_kernel(PhotoLevels L, PhotoArgs A,
                                                                  double* partials) {
  __shared__ float sref[3][kF][kF];
  __shared__ float swarp[3][kF][kF];
  __shared__ float sdep[kF][kF];
  __shared__ uint8_t sval[kF][kF];
  __shared__ double red[kPhotoSlots * kPhotoThreads];
  const Tile T = tile_of(L);
  const int l = T.l, b = T.b, h = T.h, w = T.w;
  const int tid = threadIdx.x;
  const float* depth = L.depth[l] + (size_t)b * h * w;
  for (int i = tid; i < kF * kF; i += kPhotoThreads) {
    const int rx = i % kF, ry = i / kF, gx = T.x0 - 1 + rx, gy = T.y0 - 1 + ry;
    const bool in = gx >= 0 && gy >= 0 && gx < w && gy < h;
    sdep[ry][rx] = in ? __ldg(depth + (size_t)gy * w + gx) : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) sref[c][ry][rx] = in ? image_at(A, b, 0, c, l, gx, gy) : 0.f;
  }
  const int lx = tid % kPhotoTile, ly = tid / kPhotoTile;
  const int qx = T.x0 + lx, qy = T.y0 + ly;
  const bool inside = qx < w && qy < h;
  const bool interior = inside && qx >= 1 && qy >= 1 && qx <= w - 2 && qy <= h - 2;
  const size_t hw = (size_t)h * w, qi = (size_t)qy * w + qx;
  float best_e[kPhotoMaxSources];
  int best_s[kPhotoMaxSources];
#pragma unroll
  for (int j = 0; j < kPhotoMaxSources; ++j) {
    best_e[j] = INFINITY;
    best_s[j] = -1;
  }
  int n_valid = 0;
  uint32_t valid_bits = 0;
  for (int s = 0; s < A.S; ++s) {
    float P[12];
    const float* Pg = A.proj + (((size_t)b * A.S + s) * L.levels + l) * 12;
#pragma unroll
    for (int k = 0; k < 12; ++k) P[k] = __ldg(Pg + k);
    __syncthreads();                         // previous source's tile fully read
    for (int i = tid; i < kF * kF; i += kPhotoThreads) {
      const int rx = i % kF, ry = i / kF, gx = T.x0 - 1 + rx, gy = T.y0 - 1 + ry;
      WarpPt p;
      p.ok = false;
      if (gx >= 0 && gy >= 0 && gx < w && gy < h) p = warp_point(P, gx, gy, sdep[ry][rx], w, h);
      sval[ry][rx] = p.ok;
#pragma unroll
      for (int c = 0; c < 3; ++c) swarp[c][ry][rx] = p.ok ? bilinear(taps(A, b, s, c, l, p), p) : 0.f;
    }
    __syncthreads();
    if (!inside) continue;
    bool ok = interior;
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int i = 0; i < 3; ++i) ok = ok && sval[ly + j][lx + i];
    float e = NAN;
    if (ok) {
      float ssim_sum = 0.f, l1_sum = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const WinStats st = window_stats<kF>(sref, swarp, c, lx + 1, ly + 1);
        const float a1 = fmaf(2.f * st.mx, st.my, kPhotoC1), a2 = fmaf(2.f, st.sxy, kPhotoC2);
        const float b1 = fmaf(st.mx, st.mx, fmaf(st.my, st.my, kPhotoC1));
        const float b2 = st.sxx + st.syy + kPhotoC2;
        ssim_sum += __fdiv_rn(a1 * a2, b1 * b2);
        l1_sum += fabsf(sref[c][ly + 1][lx + 1] - swarp[c][ly + 1][lx + 1]);
      }
      e = fmaf(kPhotoAlpha * 0.5f, (3.f - ssim_sum) * (1.f / 3.f), (1.f - kPhotoAlpha) * l1_sum * (1.f / 3.f));
      // a non-finite e (non-finite input) cannot be ordered: the pair counts as not valid, so
      // every one of the n_valid entries below is in the sorted list
      ok = isfinite(e);
      if (!ok) e = NAN;
    }
    if (ok) {
      valid_bits |= 1u << s;
      ++n_valid;
      // insertion into the sorted list; sources arrive in index order, so ties keep that order
      float ce = e;
      int cs = s;
#pragma unroll
      for (int j = 0; j < kPhotoMaxSources; ++j) {
        if (ce < best_e[j]) {
          const float te = best_e[j];
          const int ts = best_s[j];
          best_e[j] = ce;
          best_s[j] = cs;
          ce = te;
          cs = ts;
        }
      }
    }
    if (L.dbg_e[l]) L.dbg_e[l][((size_t)b * A.S + s) * hw + qi] = e;
  }
  const int nsel = min(A.K, n_valid);
  double loss_q = 0.0;
  uint32_t mask = 0;
#pragma unroll
  for (int j = 0; j < kPhotoMaxSources; ++j)
    if (j < nsel) {
      loss_q += (double)best_e[j];
      mask |= 1u << best_s[j];
    }
  if (nsel) loss_q /= nsel;
  double v[kPhotoSlots] = {loss_q, nsel ? 1.0 : 0.0, 0.0, 0.0};
  if (inside) {
    L.sel[l][(size_t)b * hw + qi] = (uint16_t)mask;
    if (L.dbg_valid[l]) L.dbg_valid[l][(size_t)b * hw + qi] = (uint16_t)valid_bits;
    if (L.dbg_lossq[l]) L.dbg_lossq[l][(size_t)b * hw + qi] = nsel ? (float)loss_q : NAN;
    const float delta = __fmul_rn(__ldg(A.dint + b), L.ratio[l]);
    const float dq = depth_hat(sdep[ly + 1][lx + 1], delta);
    if (qx + 1 < w) {
      const float g = (fabsf(sref[0][ly + 1][lx + 2] - sref[0][ly + 1][lx + 1]) +
                       fabsf(sref[1][ly + 1][lx + 2] - sref[1][ly + 1][lx + 1]) +
                       fabsf(sref[2][ly + 1][lx + 2] - sref[2][ly + 1][lx + 1])) * (1.f / 3.f);
      v[2] = (double)(fabsf(depth_hat(sdep[ly + 1][lx + 2], delta) - dq) * expf(-g));
    }
    if (qy + 1 < h) {
      const float g = (fabsf(sref[0][ly + 2][lx + 1] - sref[0][ly + 1][lx + 1]) +
                       fabsf(sref[1][ly + 2][lx + 1] - sref[1][ly + 1][lx + 1]) +
                       fabsf(sref[2][ly + 2][lx + 1] - sref[2][ly + 1][lx + 1])) * (1.f / 3.f);
      v[3] = (double)(fabsf(depth_hat(sdep[ly + 2][lx + 1], delta) - dq) * expf(-g));
    }
  }
  photo_block_reduce(v, red);
  if (tid < kPhotoSlots) partials[(size_t)tid * gridDim.x + blockIdx.x] = red[tid * kPhotoThreads];
}

// One block: per level, each slot's block partials in a fixed order -> loss, stats (P_l, S_l,
// N_l as float32) and counts (N_l, int64, for the backward).
__global__ void __launch_bounds__(kPhotoThreads) photo_finish_kernel(PhotoLevels L, PhotoArgs A,
                                                                     const double* partials, int nblocks,
                                                                     float* loss, float* stats,
                                                                     long long* counts) {
  __shared__ double red[kPhotoSlots * kPhotoThreads];
  double total = 0.0;
  for (int l = 0; l < L.levels; ++l) {
    double v[kPhotoSlots];
#pragma unroll
    for (int s = 0; s < kPhotoSlots; ++s) {
      double acc = 0.0;
      for (int k = L.begin[l] + threadIdx.x; k < L.begin[l + 1]; k += kPhotoThreads)
        acc += partials[(size_t)s * nblocks + k];
      v[s] = acc;
    }
    photo_block_reduce(v, red);
    const double n = red[kPhotoThreads];
    const double P = n > 0.0 ? red[0] / n : 0.0;
    const double h = L.h[l], w = L.w[l];
    const double S = red[2 * kPhotoThreads] / (A.B * h * (w - 1)) + red[3 * kPhotoThreads] / (A.B * (h - 1) * w);
    total += ldexp(1.0, 1 - l) * (P + (double)A.lambda * S);
    if (threadIdx.x == 0) {
      stats[3 * l] = (float)P;
      stats[3 * l + 1] = (float)S;
      stats[3 * l + 2] = (float)n;
      counts[l] = (long long)n;
    }
    __syncthreads();                       // red is reused by the next level
  }
  if (threadIdx.x == 0) *loss = (float)total;
}

__global__ void __launch_bounds__(kPhotoThreads) photo_bwd_kernel(PhotoLevels L, PhotoArgs A,
                                                                  const long long* counts,
                                                                  const float* grad_loss) {
  __shared__ float sref[3][kG][kG];
  __shared__ float swarp[3][kG][kG];
  __shared__ uint8_t sval[kG][kG];
  __shared__ float sdep[kG][kG];
  __shared__ float scoef[kF][kF][12];    // per window q: (a, b, c) per channel, then the L1 terms
  const Tile T = tile_of(L);
  const int l = T.l, b = T.b, h = T.h, w = T.w;
  const int tid = threadIdx.x;
  const size_t hw = (size_t)h * w;
  const float* depth = L.depth[l] + (size_t)b * hw;
  const uint16_t* sel = L.sel[l] + (size_t)b * hw;
  for (int i = tid; i < kG * kG; i += kPhotoThreads) {
    const int rx = i % kG, ry = i / kG, gx = T.x0 - 2 + rx, gy = T.y0 - 2 + ry;
    const bool in = gx >= 0 && gy >= 0 && gx < w && gy < h;
    sdep[ry][rx] = in ? __ldg(depth + (size_t)gy * w + gx) : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) sref[c][ry][rx] = in ? image_at(A, b, 0, c, l, gx, gy) : 0.f;
  }
  __syncthreads();       // the smoothness terms read the staged tile even when no source runs
  const float gl = __fmul_rn(__ldg(grad_loss), (float)ldexp(1.0, 1 - l));
  const long long n_l = counts[l];
  const float gscale = n_l > 0 ? (float)((double)gl / (double)n_l) : 0.f;
  const int lx = tid % kPhotoTile, ly = tid / kPhotoTile;
  const int px = T.x0 + lx, py = T.y0 + ly;
  const bool inside = px < w && py < h;
  float grad = 0.f;
  for (int s = 0; s < A.S && gscale != 0.f; ++s) {
    float P[12];
    const float* Pg = A.proj + (((size_t)b * A.S + s) * L.levels + l) * 12;
#pragma unroll
    for (int k = 0; k < 12; ++k) P[k] = __ldg(Pg + k);
    __syncthreads();
    for (int i = tid; i < kG * kG; i += kPhotoThreads) {
      const int rx = i % kG, ry = i / kG, gx = T.x0 - 2 + rx, gy = T.y0 - 2 + ry;
      WarpPt p;
      p.ok = false;
      if (gx >= 0 && gy >= 0 && gx < w && gy < h) p = warp_point(P, gx, gy, sdep[ry][rx], w, h);
      sval[ry][rx] = p.ok;
#pragma unroll
      for (int c = 0; c < 3; ++c) swarp[c][ry][rx] = p.ok ? bilinear(taps(A, b, s, c, l, p), p) : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < kF * kF; i += kPhotoThreads) {
      const int rx = i % kF, ry = i / kF, gx = T.x0 - 1 + rx, gy = T.y0 - 1 + ry;
      float* co = scoef[ry][rx];
      const uint32_t m = (gx >= 1 && gy >= 1 && gx <= w - 2 && gy <= h - 2) ? sel[(size_t)gy * w + gx] : 0u;
      if (!((m >> s) & 1u)) {
#pragma unroll
        for (int k = 0; k < 12; ++k) co[k] = 0.f;
        continue;
      }
      const float k_q = gscale / (float)__popc(m);
      const float k_ssim = k_q * (kPhotoAlpha / 3.f) * -0.5f;
      const float k_l1 = k_q * ((1.f - kPhotoAlpha) / 3.f);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const WinStats st = window_stats<kG>(sref, swarp, c, rx + 1, ry + 1);
        const float a1 = fmaf(2.f * st.mx, st.my, kPhotoC1), a2 = fmaf(2.f, st.sxy, kPhotoC2);
        const float b1 = fmaf(st.mx, st.mx, fmaf(st.my, st.my, kPhotoC1));
        const float b2 = st.sxx + st.syy + kPhotoC2;
        const float ssim = __fdiv_rn(a1 * a2, b1 * b2);
        const float ib = __frcp_rn(b1 * b2);
        // dSSIM/dy_i = a + b x_i + c y_i over the window's 9 samples
        const float ca = (2.f / 9.f) * (st.mx * a2 * ib - st.my * ssim / b1 - st.mx * a1 * ib + st.my * ssim / b2);
        const float cb = (2.f / 9.f) * a1 * ib;
        const float cc = -(2.f / 9.f) * ssim / b2;
        co[3 * c] = k_ssim * ca;
        co[3 * c + 1] = k_ssim * cb;
        co[3 * c + 2] = k_ssim * cc;
        co[9 + c] = -k_l1 * sgnf(sref[c][ry + 1][rx + 1] - swarp[c][ry + 1][rx + 1]);
      }
    }
    __syncthreads();
    if (!inside || !sval[ly + 2][lx + 2]) continue;
    float G[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float xv = sref[c][ly + 2][lx + 2], yv = swarp[c][ly + 2][lx + 2];
      float g = scoef[ly + 1][lx + 1][9 + c];
#pragma unroll
      for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const float* co = scoef[ly + j][lx + i];
          g += co[3 * c] + co[3 * c + 1] * xv + co[3 * c + 2] * yv;
        }
      G[c] = g;
    }
    if (G[0] == 0.f && G[1] == 0.f && G[2] == 0.f) continue;
    const float d = sdep[ly + 2][lx + 2];
    const WarpPt p = warp_point(P, px, py, d, w, h);
    // du/dd = (u T_z - T_x) / (d^2 p_z), dv/dd likewise (p = R (x, y, 1) + T / d)
    const float k = p.inv_d * p.inv_d / p.pz;
    const float dudd = (p.u * P[11] - P[3]) * k, dvdd = (p.v * P[11] - P[7]) * k;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const Taps4 t = taps(A, b, s, c, l, p);
      const float dydu = fmaf(p.fy, t.v11 - t.v10, (1.f - p.fy) * (t.v01 - t.v00));
      const float dydv = fmaf(p.fx, t.v11 - t.v01, (1.f - p.fx) * (t.v10 - t.v00));
      grad = fmaf(G[c], fmaf(dydu, dudd, dydv * dvdd), grad);
    }
  }
  if (!inside) return;
  // smoothness: the pairs (p-1, p), (p, p+1) in x and in y
  const float delta = __fmul_rn(__ldg(A.dint + b), L.ratio[l]);
  const float ks = gl * A.lambda / delta;
  const int cx = lx + 2, cy = ly + 2;
  const float dp = depth_hat(sdep[cy][cx], delta);
  auto edge = [&](int ax, int ay, int bx, int by) {   // exp(-g) between staged pixels a and b
    const float g = (fabsf(sref[0][by][bx] - sref[0][ay][ax]) + fabsf(sref[1][by][bx] - sref[1][ay][ax]) +
                     fabsf(sref[2][by][bx] - sref[2][ay][ax])) * (1.f / 3.f);
    return expf(-g);
  };
  float sm = 0.f;
  if (w > 1) {
    const float nx = (float)((double)A.B * h * (w - 1));
    if (px >= 1) sm += sgnf(dp - depth_hat(sdep[cy][cx - 1], delta)) * edge(cx - 1, cy, cx, cy) / nx;
    if (px + 1 < w) sm -= sgnf(depth_hat(sdep[cy][cx + 1], delta) - dp) * edge(cx, cy, cx + 1, cy) / nx;
  }
  if (h > 1) {
    const float ny = (float)((double)A.B * (h - 1) * w);
    if (py >= 1) sm += sgnf(dp - depth_hat(sdep[cy - 1][cx], delta)) * edge(cx, cy - 1, cx, cy) / ny;
    if (py + 1 < h) sm -= sgnf(depth_hat(sdep[cy + 1][cx], delta) - dp) * edge(cx, cy, cx, cy + 1) / ny;
  }
  L.grad[l][(size_t)b * hw + (size_t)py * w + px] = fmaf(ks, sm, grad);
}

static int make_photo_levels(PhotoLevels& L, PhotoArgs& A, const float* imgs, const float* proj,
                             const float* dint, const float* const* depth, const float* ratios, int B,
                             int V, int H, int W, int levels, int K, float lambda, const char* what) {
  CASMVS_REQUIRE(imgs && proj && dint && depth && ratios, "%s: null pointer", what);
  CASMVS_REQUIRE(levels >= 1 && levels <= kPhotoMaxLevels, "%s: levels must be in 1..%d", what,
                 kPhotoMaxLevels);
  const int S = V - 1;
  CASMVS_REQUIRE(S >= 1 && S <= kPhotoMaxSources, "%s: %d source views; 1..%d are supported", what, S,
                 kPhotoMaxSources);
  CASMVS_REQUIRE(K >= 1 && K <= S, "%s: top-K %d must be in 1..%d (the source count)", what, K, S);
  CASMVS_REQUIRE(B >= 1, "%s: bad batch %d", what, B);
  CASMVS_REQUIRE(isfinite(lambda) && lambda >= 0.f, "%s: smoothness weight must be finite and >= 0",
                 what);
  const int div = 1 << (levels - 1);
  CASMVS_REQUIRE(H % div == 0 && W % div == 0, "%s: %dx%d is not divisible by 2^%d", what, W, H,
                 levels - 1);
  L.levels = levels;
  L.begin[0] = 0;
  long long blocks = 0;
  for (int l = 0; l < levels; ++l) {
    CASMVS_REQUIRE(depth[l], "%s: null depth (level %d)", what, l);
    CASMVS_REQUIRE(ratios[l] > 0.f, "%s: interval ratio of level %d must be > 0", what, l);
    L.h[l] = H >> l;
    L.w[l] = W >> l;
    CASMVS_REQUIRE(L.h[l] >= 3 && L.w[l] >= 3, "%s: level %d is %dx%d, smaller than 3x3", what, l,
                   L.w[l], L.h[l]);
    L.depth[l] = depth[l];
    L.ratio[l] = ratios[l];
    L.tiles_x[l] = (L.w[l] + kPhotoTile - 1) / kPhotoTile;
    L.tiles_y[l] = (L.h[l] + kPhotoTile - 1) / kPhotoTile;
    blocks += (long long)L.tiles_x[l] * L.tiles_y[l] * B;
    CASMVS_REQUIRE(blocks < (1ll << 30), "%s: too many tiles", what);
    L.begin[l + 1] = (int)blocks;
    L.grad[l] = nullptr;
    L.sel[l] = nullptr;
    L.dbg_e[l] = nullptr;
    L.dbg_valid[l] = nullptr;
    L.dbg_lossq[l] = nullptr;
  }
  A.imgs = imgs;
  A.proj = proj;
  A.dint = dint;
  A.B = B;
  A.S = S;
  A.H = H;
  A.W = W;
  A.K = K;
  A.lambda = lambda;
  return 0;
}

static long long photo_blocks(int B, int H, int W, int levels) {
  long long n = 0;
  for (int l = 0; l < levels && l < kPhotoMaxLevels; ++l)
    n += (long long)(((W >> l) + kPhotoTile - 1) / kPhotoTile) * (((H >> l) + kPhotoTile - 1) / kPhotoTile) * B;
  return n;
}

}  // namespace casmvs

using namespace casmvs;

extern "C" size_t casmvs_photo_loss_workspace_bytes(int B, int H, int W, int levels) {
  if (B < 1 || H < 1 || W < 1 || levels < 1) return 0;
  return (size_t)kPhotoSlots * photo_blocks(B, H, W, levels) * sizeof(double);
}

extern "C" int casmvs_photo_loss_fwd(const float* imgs, const float* proj_mats, const float* depth_interval,
                                     const float* const* depth, const float* interval_ratios, int B, int V,
                                     int H, int W, int levels, int topk, float smooth_weight,
                                     uint16_t* const* selection, float* loss, float* stats,
                                     long long* counts, float* const* dbg_e, uint16_t* const* dbg_valid,
                                     float* const* dbg_lossq, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  PhotoLevels L;
  PhotoArgs A;
  if (int rc = make_photo_levels(L, A, imgs, proj_mats, depth_interval, depth, interval_ratios, B, V, H, W,
                                 levels, topk, smooth_weight, "photo_loss_fwd"))
    return rc;
  CASMVS_REQUIRE(selection && loss && stats && counts, "photo_loss_fwd: null output");
  for (int l = 0; l < levels; ++l) {
    CASMVS_REQUIRE(selection[l], "photo_loss_fwd: null selection (level %d)", l);
    L.sel[l] = selection[l];
    L.dbg_e[l] = dbg_e ? dbg_e[l] : nullptr;
    L.dbg_valid[l] = dbg_valid ? dbg_valid[l] : nullptr;
    L.dbg_lossq[l] = dbg_lossq ? dbg_lossq[l] : nullptr;
  }
  const size_t need = casmvs_photo_loss_workspace_bytes(B, H, W, levels);
  CASMVS_REQUIRE(workspace && workspace_bytes >= need, "photo_loss_fwd: workspace too small (%zu B needed)",
                 need);
  cudaStream_t st = as_stream(stream);
  const int nblocks = L.begin[levels];
  double* partials = static_cast<double*>(workspace);
  photo_fwd_kernel<<<nblocks, kPhotoThreads, 0, st>>>(L, A, partials);
  if (int rc = after_launch("photo_fwd")) return rc;
  photo_finish_kernel<<<1, kPhotoThreads, 0, st>>>(L, A, partials, nblocks, loss, stats, counts);
  return after_launch("photo_finish");
}

extern "C" int casmvs_photo_loss_bwd(const float* imgs, const float* proj_mats, const float* depth_interval,
                                     const float* const* depth, const float* interval_ratios, int B, int V,
                                     int H, int W, int levels, int topk, float smooth_weight,
                                     const uint16_t* const* selection, const long long* counts,
                                     const float* grad_loss, float* const* grad_depth, void* stream) {
  PhotoLevels L;
  PhotoArgs A;
  if (int rc = make_photo_levels(L, A, imgs, proj_mats, depth_interval, depth, interval_ratios, B, V, H, W,
                                 levels, topk, smooth_weight, "photo_loss_bwd"))
    return rc;
  CASMVS_REQUIRE(selection && counts && grad_loss && grad_depth, "photo_loss_bwd: null pointer");
  for (int l = 0; l < levels; ++l) {
    CASMVS_REQUIRE(selection[l] && grad_depth[l], "photo_loss_bwd: null pointer (level %d)", l);
    L.sel[l] = const_cast<uint16_t*>(selection[l]);
    L.grad[l] = grad_depth[l];
  }
  photo_bwd_kernel<<<L.begin[levels], kPhotoThreads, 0, as_stream(stream)>>>(L, A, counts, grad_loss);
  return after_launch("photo_loss_bwd");
}
