// K1, TMA-staged generation — fused homography plane-sweep warp + bilinear sample + variance
// with the source-view footprints of a pixel tile staged in shared memory.
//
// Replaces (reference, paths relative to /root/reference):
//   homo_warp                      models/modules.py:52-92   (called V-1 times)
//   variance accumulation          models/mvsnet.py:137-141,147-156,166-168
//
// Why: the gather-from-L1 kernel (warp_cost.cu) fetches 4 taps x (V-1) views per output
// through the L1 tag stage and leaves every L1 miss to the several-hundred-cycle L2 round
// trip, so it stalls on long-scoreboard waits well below the HBM bound.  Here a
// CTA owns a TW x TH tile of reference pixels x a run of depth planes:
//   1. every thread evaluates its sample position in each source view at the first and last
//      plane of the run (positions are monotonic along the epipolar line in 1/depth), a block
//      min/max gives the footprint's bounding box per view;
//   2. ONE elected thread issues one cp.async.bulk.tensor.4d per view: box {C, BW, BH, 1} of
//      the channels-last feature map viewed as {C, w, h, B*V}, swizzle = texel bytes, landing
//      on an mbarrier.  Out-of-image texels are zero-filled by the TMA unit, which IS
//      grid_sample's zero padding: the fast path needs no border logic at all;
//   3. threads blend from shared memory (fixed ~30-cycle latency, conflict-free thanks to the
//      hardware swizzle: a quarter-warp's eight 16-byte reads land on 32 distinct banks) and
//      keep a view's 2x2 window in registers while it does not move between planes (the sweep
//      advances ~0.4 texel per plane in the cascade, so >half of the window loads vanish);
//   4. a sample whose window is not inside the staged box (depth discontinuity inside the
//      tile, exotic geometry) takes the robust gather path for that sample only; if the
//      footprint of the whole run does not fit, the CTA halves the run and stages again.
// The warped (B,V-1,C,D,h,w) volumes never exist; features are read from L2 once per
// (tile, run), hypotheses once, the cost volume is written once, 32 bytes per thread as two 16-byte stores.
#include <limits.h>

#include "k1_common.cuh"
#include "tma_common.cuh"

namespace casmvs {
namespace k1s {

using tc::fence_barrier_init;
using tc::mbar_init;
using tc::mbar_wait;
using tc::smem_u32;

constexpr int kMaxSrcSmem = 2;
constexpr int kMarginX = 16, kMarginY = 4;    // box = tile + margins (see launch)
constexpr float kMagic = 12582912.f;          // 1.5 * 2^23: u + kMagic (round down) = floor(u) + kMagic
constexpr int kMagicBits = 0x4B400000;

__device__ __forceinline__ float fadd_rd(float a, float b) { return __fadd_rd(a, b); }

template <int TEXB>
__device__ __forceinline__ uint32_t swz(uint32_t off) {   // off: bytes from a 1024 B-aligned base
  constexpr uint32_t m = (TEXB == 128 ? 7u : TEXB == 64 ? 3u : 1u) << 4;
  return off ^ ((off >> 3) & m);
}
__device__ __forceinline__ void lds_tex(uint32_t addr, Tex8& t) {   // 2 x 16 B, second half at ^16
  asm volatile("ld.shared.v2.b64 {%0,%1}, [%2];" : "=l"(t.v[0]), "=l"(t.v[1]) : "r"(addr));
  asm volatile("ld.shared.v2.b64 {%0,%1}, [%2];" : "=l"(t.v[2]), "=l"(t.v[3]) : "r"(addr ^ 16u));
}

struct Small {            // lives behind the boxes in dynamic shared memory
  float proj[kMaxSrcSmem * 12];
  int mm[kMaxSrcSmem * 4];      // minx, miny, maxx, maxy per view (block reduction)
  unsigned long long bar;
};

// What a thread of either kernel knows after the per-CTA set-up.
template <int NSRC>
struct Tile {
  uint32_t base;            // 1024 B-aligned start of the boxes (shared-window address)
  uint32_t bar;             // the CTA's mbarrier
  Small* sm;
  int sub, c0, pix;         // channel group of this thread, its first channel, its pixel
  bool active;              // the pixel is inside the image
  float ax[NSRC], ay[NSRC], az[NSRC], tx[NSRC], ty[NSRC], tz[NSRC];   // R*(x,y,1) and T per view
};

// Tile coordinates, projection rows of the NSRC source views into Small, mbarrier init, and
// the per-view terms of the homography at this thread's pixel.
template <int NSRC, int TW, int TH, int TPP>
__device__ __forceinline__ Tile<NSRC> setup_tile(uint8_t* smem_raw, const float* __restrict__ proj,
                                                 int h, int w, int box_stride, int tiles_x) {
  Tile<NSRC> t;
  t.base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  t.sm = reinterpret_cast<Small*>(smem_raw + (t.base - smem_u32(smem_raw)) + NSRC * box_stride);
  t.bar = smem_u32(&t.sm->bar);
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int tile_y = blockIdx.x / tiles_x, tile_x = blockIdx.x - tile_y * tiles_x;
  const int lp = tid / TPP;
  t.sub = tid - lp * TPP;
  t.c0 = t.sub * kCPT;   // before the barrier: computed after it, ptxas spends 3-6 more registers
  const int py = lp / TW, px = lp - py * TW;
  const int xr = tile_x * TW + px, yr = tile_y * TH + py;
  t.active = xr < w && yr < h;
  const int x = min(xr, w - 1), y = min(yr, h - 1);
  t.pix = y * w + x;

  for (int i = tid; i < NSRC * 12; i += TW * TH * TPP) t.sm->proj[i] = proj[(size_t)b * NSRC * 12 + i];
  if (tid == 0) {
    mbar_init(t.bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  const float xf = (float)x, yf = (float)y;
#pragma unroll
  for (int v = 0; v < NSRC; ++v) {
    const float* P = t.sm->proj + v * 12;
    t.ax[v] = fmaf(P[0], xf, fmaf(P[1], yf, P[2]));     // R*(x,y,1)   (modules.py:72)
    t.ay[v] = fmaf(P[4], xf, fmaf(P[5], yf, P[6]));
    t.az[v] = fmaf(P[8], xf, fmaf(P[9], yf, P[10]));
    t.tx[v] = P[3]; t.ty[v] = P[7]; t.tz[v] = P[11];
  }
  return t;
}

// Footprint of planes [d0, d0 + n) in every view, n = d_end - d0 halved until every view's
// footprint fits its BW x BH box (or n == 1); then one elected thread stages the boxes, one TMA
// per view with zero fill outside the image, completing on the CTA's mbarrier.  Returns n;
// kx / ky: the box origins plus kMagicBits, for the floor-by-add of the sampling loops.
template <int NSRC, int TEXB, class HP>
__device__ __forceinline__ int stage_boxes(const Tile<NSRC>& t, const CUtensorMap& fmap,
                                           const HP& hp, int d0, int d_end, int h, int w,
                                           int BW, int BH, int box_stride, int (&kx)[NSRC],
                                           int (&ky)[NSRC]) {
  const int tid = threadIdx.x;
  Small* sm = t.sm;
  int n = d_end - d0;
  int bx[NSRC], by[NSRC];
  for (;;) {
    // (also: every thread is done with the previous run's boxes and min/max words)
    __syncthreads();
    if (tid < NSRC * 4) sm->mm[tid] = (tid & 2) ? INT_MIN : INT_MAX;
    __syncthreads();
    const float ia = rcp_approx(hp.at(d0));
    const float ib = rcp_approx(hp.at(d0 + n - 1));
#pragma unroll
    for (int v = 0; v < NSRC; ++v) {
      int mnx = INT_MAX, mny = INT_MAX, mxx = INT_MIN, mxy = INT_MIN;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float id = e ? ib : ia;
        const float qz = fmaf(t.tz[v], id, t.az[v]);
        const float rz = rcp_approx(qz);
        const float u = fmaf(t.tx[v], id, t.ax[v]) * rz, vv = fmaf(t.ty[v], id, t.ay[v]) * rz;
        // samples that cannot touch the image (or are not finite) do not shape the box
        if (t.active && qz > 1e-7f && u > -2.f && u < (float)(w + 1) && vv > -2.f &&
            vv < (float)(h + 1)) {
          const int xi = __float2int_rd(u), yi = __float2int_rd(vv);
          mnx = min(mnx, xi); mxx = max(mxx, xi);
          mny = min(mny, yi); mxy = max(mxy, yi);
        }
      }
      mnx = __reduce_min_sync(0xffffffffu, mnx); mny = __reduce_min_sync(0xffffffffu, mny);
      mxx = __reduce_max_sync(0xffffffffu, mxx); mxy = __reduce_max_sync(0xffffffffu, mxy);
      if ((tid & 31) == 0) {
        atomicMin(&sm->mm[v * 4 + 0], mnx); atomicMin(&sm->mm[v * 4 + 1], mny);
        atomicMax(&sm->mm[v * 4 + 2], mxx); atomicMax(&sm->mm[v * 4 + 3], mxy);
      }
    }
    __syncthreads();
    bool fits = true;
#pragma unroll
    for (int v = 0; v < NSRC; ++v) {
      const int mnx = sm->mm[v * 4 + 0], mny = sm->mm[v * 4 + 1];
      const int mxx = sm->mm[v * 4 + 2], mxy = sm->mm[v * 4 + 3];
      if (mnx > mxx) { bx[v] = 0; by[v] = 0; continue; }      // nothing lands in the image
      const int sx = mxx + 2 - mnx, sy = mxy + 2 - mny;       // texel columns / rows needed
      if (sx > BW || sy > BH) fits = false;
      bx[v] = mnx - max(0, (BW - sx) >> 1);
      by[v] = mny - max(0, (BH - sy) >> 1);
    }
    if (fits || n == 1) break;
    n = (n + 1) >> 1;
  }
  if (tid == 0) {
    const int b = blockIdx.y;
    tma::mbar_expect_tx(t.bar, (uint32_t)(NSRC * BW * BH * TEXB));
#pragma unroll
    for (int v = 0; v < NSRC; ++v)
      tma::tma_load_4d(t.base + v * box_stride, &fmap, t.bar, 0, bx[v], by[v], b * (NSRC + 1) + v + 1);
  }
#pragma unroll
  for (int v = 0; v < NSRC; ++v) { kx[v] = kMagicBits + bx[v]; ky[v] = kMagicBits + by[v]; }
  return n;
}

// NSRC source views, C channels, TW x TH pixel tile.  Every plane loads its 2x2 windows (the
// plane-group kernel below re-uses them); variance or 8-group correlation epilogue.
// BLOCKED: the cost volume is stored blocked by channel quads (B, COUT/4, D, h, w, 4) instead of
// channels-last.  A template parameter: as a run-time value it cost the channels-last kernels
// about 5 % of their rate.  INV: a ladder is in inverse depth (HypPixT).  PIX: a ladder has a
// per-pixel step map (the adaptive mode).  The body of warp_var_smem_kernel (uniform),
// warp_var_smem_inv_kernel and warp_var_smem_pix_kernel below.
template <int NSRC, int C, int TW, int TH, int MINB, bool GWC, bool BLOCKED, bool INV,
          bool PIX = false>
__device__ __forceinline__ void
warp_var_smem(const CUtensorMap& fmap, const float* __restrict__ feats,
              const float* __restrict__ proj, const Hyp hyp,
              float* __restrict__ cost, int D, int h, int w, int dchunk, int BW, int BH,
              int box_stride, int tiles_x, int round_tf32) {
  // GWC (group-wise correlation, mvsnet.py:143-144,158-162,170-172) is built for 8 groups:
  // C/8 in {1,2,4} channels per group, every thread owns 8/(C/8) whole groups
  constexpr int V = NSRC + 1, TPP = C / kCPT, TEXB = C * 4;
  constexpr int CPG = C / 8, NG = kCPT / CPG, COUT = GWC ? 8 : C;
  extern __shared__ uint8_t smem_raw[];
  const Tile<NSRC> t = setup_tile<NSRC, TW, TH, TPP>(smem_raw, proj, h, w, box_stride, tiles_x);
  const int b = blockIdx.y;
  const int c0 = t.c0;
  const int hw = h * w, pix = t.pix;

  const size_t view_stride = (size_t)hw * C;
  const float* fb = feats + (size_t)b * V * view_stride + c0;
  const Tex8 ref = ldg256(fb + (size_t)pix * C);
  const float inv_v = 1.f / (float)V;
  const u64 inv_v2 = pk2(inv_v, inv_v), ninv_v2 = pk2(-inv_v, -inv_v);

  const int d_begin = blockIdx.z * dchunk;
  const int d_end = min(D, d_begin + dchunk);
  const HypPixT<INV, PIX> hp(hyp, b, D, (size_t)hw, pix);
  // output: channels-last, or blocked by channel quads (B, COUT/4, D, h, w, 4)
  const int co = GWC ? t.sub * NG : c0;
  const size_t pstr = BLOCKED ? (size_t)hw * 4 : (size_t)hw * COUT;      // next plane
  const size_t qstr = BLOCKED ? (size_t)D * hw * 4 : 4;                 // next channel quad
  float* optr = cost + (BLOCKED ? (((size_t)b * (COUT / 4) + co / 4) * D + d_begin) * hw * 4 +
                                      (size_t)pix * 4 + (co & 3)
                                : ((size_t)(b * D + d_begin) * hw + pix) * COUT + co);
  const int row_b = BW * TEXB;

  uint32_t phase = 0;

  for (int d0 = d_begin; d0 < d_end;) {
    int kx[NSRC], ky[NSRC];
    const int n = stage_boxes<NSRC, TEXB>(t, fmap, hp, d0, d_end, h, w, BW, BH, box_stride, kx, ky);
    float depth_next = hp.at(d0);
    mbar_wait(t.bar, phase);
    phase ^= 1;

    // the planes of this run
    for (int d = d0; d < d0 + n; ++d) {
      const float inv_d = rcp_approx(depth_next);
      if (d + 1 < d0 + n) depth_next = hp.at(d + 1);
      u64 S[4], Q[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        S[k] = GWC ? 0ull : ref.v[k];            // gwc: the reference is NOT in the sum (:144)
        Q[k] = mul2(ref.v[k], ref.v[k]);
      }
#pragma unroll
      for (int v = 0; v < NSRC; ++v) {
        const float qx = fmaf(t.tx[v], inv_d, t.ax[v]);
        const float qy = fmaf(t.ty[v], inv_d, t.ay[v]);
        const float qz = fmaf(t.tz[v], inv_d, t.az[v]);
        const float rz = rcp_approx(qz);
        const float u = qx * rz, vv = qy * rz;
        // floor via round-down add: exact for |u| < 2^22, anything else fails the range test
        const float fu = fadd_rd(u, kMagic), fv = fadd_rd(vv, kMagic);
        const int xi = __float_as_int(fu) - kx[v], yi = __float_as_int(fv) - ky[v];
        const bool inbox = (unsigned)xi < (unsigned)(BW - 1) && (unsigned)yi < (unsigned)(BH - 1) &&
                           qz > 1e-7f;
        u64 r[4];
        const auto put_r = [&r](int k, u64 x) { r[k] = x; };
        if (__builtin_expect(inbox, 1)) {
          const float fx = u - (fu - kMagic), fy = vv - (fv - kMagic);
          const float wxa = 1.f - fx, wya = 1.f - fy;
          const int l00 = v * box_stride + yi * row_b + xi * TEXB + c0 * 4;
          Window win;
          lds_tex(t.base + swz<TEXB>(l00), win.t00);
          lds_tex(t.base + swz<TEXB>(l00 + TEXB), win.t01);
          lds_tex(t.base + swz<TEXB>(l00 + row_b), win.t10);
          lds_tex(t.base + swz<TEXB>(l00 + row_b + TEXB), win.t11);
          blend(win, wxa * wya, fx * wya, wxa * fy, fx * fy, put_r);
        } else if (qz <= 1e-7f || u <= -1.f || u >= (float)w || vv <= -1.f || vv >= (float)h) {
          // behind the camera (modules.py:76-79) or entirely outside the source image: the
          // sample is exactly zero, S and Q are unchanged
          continue;
        } else {
          // robust gather path for a window outside the staged box (NaN propagates like ATen)
          gather_sample<C>(fb + (size_t)(v + 1) * view_stride, qx, qy, qz, h, w, C, w * C, put_r);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          S[k] = add2(S[k], r[k]);
          if (!GWC) Q[k] = fma2(r[k], r[k], Q[k]);
        }
      }
      if constexpr (GWC) {
        // cost[g] = mean_{c in g}(S_c * ref_c) / (V-1)     (mvsnet.py:170-172)
        float pr[kCPT], o[NG];
#pragma unroll
        for (int k = 0; k < 4; ++k) unpk2(mul2(S[k], ref.v[k]), pr[2 * k], pr[2 * k + 1]);
#pragma unroll
        for (int k = 0; k < NG; ++k) {
          float acc = CPG == 1 ? pr[k] : CPG == 2 ? pr[2 * k] + pr[2 * k + 1]
                      : (pr[4 * k] + pr[4 * k + 1]) + (pr[4 * k + 2] + pr[4 * k + 3]);
          float val = __fdiv_rn(acc * (1.f / (float)CPG), (float)NSRC);
          o[k] = round_tf32 ? round_tf32_f(val) : val;
        }
        if (t.active) {
          if constexpr (NG == 8) {
            u64 ov[4] = {pk2(o[0], o[1]), pk2(o[2], o[3]), pk2(o[4], o[5]), pk2(o[6], o[7])};
            stg256q(optr, qstr, ov);
          } else if constexpr (NG == 4) {
            st4(optr, make_float4(o[0], o[1], o[2], o[3]));
          } else {
            *reinterpret_cast<float2*>(optr) = make_float2(o[0], o[1]);
          }
        }
      } else {
        u64 o[4];
        variance(S, Q, inv_v2, ninv_v2, round_tf32, o);
        if (t.active) stg256q(optr, qstr, o);
      }
      optr += pstr;
    }
    d0 += n;
  }
}

template <int NSRC, int C, int TW, int TH, int MINB, bool GWC, bool BLOCKED>
__global__ void __launch_bounds__(TW* TH*(C / kCPT), MINB)
warp_var_smem_kernel(const __grid_constant__ CUtensorMap fmap, const float* __restrict__ feats,
                     const float* __restrict__ proj, const Hyp hyp, float* __restrict__ cost, int D,
                     int h, int w, int dchunk, int BW, int BH, int box_stride, int tiles_x,
                     int round_tf32) {
  warp_var_smem<NSRC, C, TW, TH, MINB, GWC, BLOCKED, false>(
      fmap, feats, proj, hyp, cost, D, h, w, dchunk, BW, BH, box_stride, tiles_x, round_tf32);
}
template <int NSRC, int C, int TW, int TH, int MINB, bool GWC, bool BLOCKED>
__global__ void __launch_bounds__(TW* TH*(C / kCPT), MINB)
warp_var_smem_inv_kernel(const __grid_constant__ CUtensorMap fmap, const float* __restrict__ feats,
                         const float* __restrict__ proj, const Hyp hyp, float* __restrict__ cost,
                         int D, int h, int w, int dchunk, int BW, int BH, int box_stride,
                         int tiles_x, int round_tf32) {
  warp_var_smem<NSRC, C, TW, TH, MINB, GWC, BLOCKED, true>(
      fmap, feats, proj, hyp, cost, D, h, w, dchunk, BW, BH, box_stride, tiles_x, round_tf32);
}
template <int NSRC, int C, int TW, int TH, int MINB, bool GWC, bool BLOCKED>
__global__ void __launch_bounds__(TW* TH*(C / kCPT), MINB)
warp_var_smem_pix_kernel(const __grid_constant__ CUtensorMap fmap, const float* __restrict__ feats,
                         const float* __restrict__ proj, const Hyp hyp, float* __restrict__ cost,
                         int D, int h, int w, int dchunk, int BW, int BH, int box_stride,
                         int tiles_x, int round_tf32) {
  warp_var_smem<NSRC, C, TW, TH, MINB, GWC, BLOCKED, false, true>(
      fmap, feats, proj, hyp, cost, D, h, w, dchunk, BW, BH, box_stride, tiles_x, round_tf32);
}

// ---- plane-group variant: window reuse WITHOUT persistent registers -----------------------------
// Both K1 generations are bound by the LSU data pipe (32 B of tap traffic per output float),
// not by latency.  Keeping the 2x2 windows of both views in registers across planes
// cuts the shared-memory wavefronts but needs far more registers (or spills,
// whose local-memory traffic goes through the same LSU pipe).  Here a thread walks PG planes
// of ONE view before turning to the next view: the window lives only inside that short walk
// (32 registers, re-loaded only when it moves: ~0.43 texel per plane in the cascade), and what
// persists between the views is one blended value per (plane, channel) -- 8 registers per plane.
// 2 source views, variance cost.  out = (ref^2 + r1^2 + r2^2)/3 - ((ref + r1 + r2)/3)^2, summed
// in the order of the kernel above (bit-identical).
template <int C, int TW, int TH, int PG, int MINB, bool BLOCKED, bool INV, bool PIX = false>
__device__ __forceinline__ void
warp_var_smem_pg(const CUtensorMap& fmap, const float* __restrict__ feats,
                 const float* __restrict__ proj, const Hyp hyp, float* __restrict__ cost,
                 int D, int h, int w, int dchunk, int BW, int BH, int box_stride, int tiles_x,
                 int round_tf32) {
  constexpr int NSRC = 2, V = 3, TPP = C / kCPT, TEXB = C * 4;
  extern __shared__ uint8_t smem_raw[];
  const Tile<NSRC> t = setup_tile<NSRC, TW, TH, TPP>(smem_raw, proj, h, w, box_stride, tiles_x);
  const int b = blockIdx.y;
  const int c0 = t.c0;
  const int hw = h * w, pix = t.pix;
  const size_t view_stride = (size_t)hw * C;
  const float* fb = feats + (size_t)b * V * view_stride + c0;
  const Tex8 ref = ldg256(fb + (size_t)pix * C);
  const float inv_v = 1.f / (float)V;
  const u64 inv_v2 = pk2(inv_v, inv_v), ninv_v2 = pk2(-inv_v, -inv_v);
  const int d_begin = blockIdx.z * dchunk;
  const int d_end = min(D, d_begin + dchunk);
  const HypPixT<INV, PIX> hp(hyp, b, D, (size_t)hw, pix);
  // output: channels-last, or blocked by channel quads (B, C/4, D, h, w, 4)
  const size_t pstr = BLOCKED ? (size_t)hw * 4 : (size_t)hw * C;        // next plane
  const size_t qstr = BLOCKED ? (size_t)D * hw * 4 : 4;                 // next channel quad
  float* optr = cost + (BLOCKED ? (((size_t)b * (C / 4) + c0 / 4) * D + d_begin) * hw * 4 +
                                      (size_t)pix * 4
                                : ((size_t)(b * D + d_begin) * hw + pix) * C + c0);
  const int row_b = BW * TEXB;
  // a row pitch that is a multiple of 1024 B leaves the swizzle bits of an address unchanged:
  // the second window row is then the first one + row_b (launch picks BW accordingly)
  const bool rowal = (row_b & 1023) == 0;
  u64 refsq[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) refsq[k] = mul2(ref.v[k], ref.v[k]);
  uint32_t phase = 0;

  for (int d0 = d_begin; d0 < d_end;) {
    int kx[NSRC], ky[NSRC];
    const int n = stage_boxes<NSRC, TEXB>(t, fmap, hp, d0, d_end, h, w, BW, BH, box_stride, kx, ky);
    // hypotheses of the next plane group are fetched while the current one is processed
    float dnext[PG];
#pragma unroll
    for (int p = 0; p < PG; ++p) dnext[p] = hp.at(min(d0 + p, d0 + n - 1));
    mbar_wait(t.bar, phase);
    phase ^= 1;

    for (int d = d0; d < d0 + n; d += PG) {
      float inv_d[PG];
#pragma unroll
      for (int p = 0; p < PG; ++p) {
        inv_d[p] = rcp_approx(dnext[p]);
        dnext[p] = hp.at(min(d + PG + p, d0 + n - 1));
      }
      u64 r1[PG][4];
#pragma unroll
      for (int v = 0; v < NSRC; ++v) {
        Window win;
        int cur = -1;                                   // window held in win
#pragma unroll
        for (int p = 0; p < PG; ++p) {
          const float qx = fmaf(t.tx[v], inv_d[p], t.ax[v]);
          const float qy = fmaf(t.ty[v], inv_d[p], t.ay[v]);
          const float qz = fmaf(t.tz[v], inv_d[p], t.az[v]);
          const float rz = rcp_approx(qz);
          const float u = qx * rz, vv = qy * rz;
          const float fu = fadd_rd(u, kMagic), fv = fadd_rd(vv, kMagic);
          const int xi = __float_as_int(fu) - kx[v], yi = __float_as_int(fv) - ky[v];
          const bool inbox = (unsigned)xi < (unsigned)(BW - 1) && (unsigned)yi < (unsigned)(BH - 1) &&
                             qz > 1e-7f;
          u64 r[4] = {0ull, 0ull, 0ull, 0ull};          // packed +0.f: a sample that is exactly zero
          const auto put_r = [&r](int k, u64 x) { r[k] = x; };
          if (__builtin_expect(inbox, 1)) {
            const float fx = u - (fu - kMagic), fy = vv - (fv - kMagic);
            const float wxa = 1.f - fx, wya = 1.f - fy;
            const int l00 = v * box_stride + yi * row_b + xi * TEXB + c0 * 4;
            if (l00 != cur) {
              const uint32_t a0 = t.base + swz<TEXB>(l00), a1 = t.base + swz<TEXB>(l00 + TEXB);
              lds_tex(a0, win.t00);
              lds_tex(a1, win.t01);
              lds_tex(rowal ? a0 + row_b : t.base + swz<TEXB>(l00 + row_b), win.t10);
              lds_tex(rowal ? a1 + row_b : t.base + swz<TEXB>(l00 + row_b + TEXB), win.t11);
              cur = l00;
            }
            blend(win, wxa * wya, fx * wya, wxa * fy, fx * fy, put_r);
          } else if (!(qz <= 1e-7f || u <= -1.f || u >= (float)w || vv <= -1.f || vv >= (float)h)) {
            gather_sample<C>(fb + (size_t)(v + 1) * view_stride, qx, qy, qz, h, w, C, w * C, put_r);
          }
          if (v == 0) {
#pragma unroll
            for (int k = 0; k < 4; ++k) r1[p][k] = r[k];
          } else if (d + p < d0 + n) {
            // S = (ref + r1) + r2, Q = fma(r2, r2, fma(r1, r1, ref^2))
            u64 S[4], Q[4], o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              S[k] = add2(add2(ref.v[k], r1[p][k]), r[k]);
              Q[k] = fma2(r[k], r[k], fma2(r1[p][k], r1[p][k], refsq[k]));
            }
            variance(S, Q, inv_v2, ninv_v2, round_tf32, o);
            if (t.active) stg256q(optr + p * pstr, qstr, o);
          }
        }
      }
      optr += PG * pstr;
    }
    optr -= (((n + PG - 1) / PG) * PG - n) * pstr;      // a short last group advanced too far
    d0 += n;
  }
}

template <int C, int TW, int TH, int PG, int MINB, bool BLOCKED>
__global__ void __launch_bounds__(TW* TH*(C / kCPT), MINB)
warp_var_smem_pg_kernel(const __grid_constant__ CUtensorMap fmap, const float* __restrict__ feats,
                        const float* __restrict__ proj, const Hyp hyp, float* __restrict__ cost,
                        int D, int h, int w, int dchunk, int BW, int BH, int box_stride, int tiles_x,
                        int round_tf32) {
  warp_var_smem_pg<C, TW, TH, PG, MINB, BLOCKED, false>(
      fmap, feats, proj, hyp, cost, D, h, w, dchunk, BW, BH, box_stride, tiles_x, round_tf32);
}
template <int C, int TW, int TH, int PG, int MINB, bool BLOCKED>
__global__ void __launch_bounds__(TW* TH*(C / kCPT), MINB)
warp_var_smem_pg_inv_kernel(const __grid_constant__ CUtensorMap fmap,
                            const float* __restrict__ feats, const float* __restrict__ proj,
                            const Hyp hyp, float* __restrict__ cost, int D, int h, int w,
                            int dchunk, int BW, int BH, int box_stride, int tiles_x,
                            int round_tf32) {
  warp_var_smem_pg<C, TW, TH, PG, MINB, BLOCKED, true>(
      fmap, feats, proj, hyp, cost, D, h, w, dchunk, BW, BH, box_stride, tiles_x, round_tf32);
}
template <int C, int TW, int TH, int PG, int MINB, bool BLOCKED>
__global__ void __launch_bounds__(TW* TH*(C / kCPT), MINB)
warp_var_smem_pg_pix_kernel(const __grid_constant__ CUtensorMap fmap,
                            const float* __restrict__ feats, const float* __restrict__ proj,
                            const Hyp hyp, float* __restrict__ cost, int D, int h, int w,
                            int dchunk, int BW, int BH, int box_stride, int tiles_x,
                            int round_tf32) {
  warp_var_smem_pg<C, TW, TH, PG, MINB, BLOCKED, false, true>(
      fmap, feats, proj, hyp, cost, D, h, w, dchunk, BW, BH, box_stride, tiles_x, round_tf32);
}

// ---- host side -------------------------------------------------------------------------------
// The features (BV, h, w, C) as {C, w, h, BV}, box {C, BW, BH, 1}, swizzle C*4 bytes.
static int feature_map(CUtensorMap* out, const float* feats, int BV, int h, int w, int C, int BW,
                       int BH) {
  const uint64_t c = C, x = w, y = h, n = BV;
  const uint32_t bw = BW, bh = BH, bc = C;
  const tma::MapDesc d{feats, 4, C * 4, {c, x, y, n, 0}, {4 * c, 4 * c * x, 4 * c * x * y, 0},
                       {bc, bw, bh, 1, 0}, {1, 1, 1, 1, 0}};
  return tma::encode_map(d, out);
}

// One launcher for both kernels: NSRC source views, TW x TH pixel tiles.  PG > 0 launches the
// plane-group kernel, whose box row is rounded up to a multiple of 1024 B (see rowal).  form: the
// ladder form (LadderForm), which picks the uniform, _inv or _pix instantiation.
template <int NSRC, int C, int TW, int TH, int MINB, bool GWC, int PG>
static int launch(const float* feats, const float* proj, const Hyp& dv, float* cost, int B, int D,
                  int h, int w, int rnd, int blocked, int form, cudaStream_t st) {
  constexpr int NT = TW * TH * (C / kCPT);
  // box = tile + margins: sweep of the depth run + scale/rotation of the view + the 2x2 window
  constexpr int wq = PG > 0 ? 1024 / (C * 4) : 1;
  constexpr int BW = (TW + kMarginX + wq - 1) / wq * wq, BH = TH + kMarginY;
  constexpr int box_stride = (BW * BH * C * 4 + 1023) & ~1023;
  constexpr size_t smem = (size_t)NSRC * box_stride + sizeof(Small) + 1024;
  static_assert(smem <= 200 * 1024, "shared memory budget");
  auto kfn = [blocked, form] {
    if constexpr (PG > 0) {
      if (form == kLadderPixelStep)
        return blocked ? warp_var_smem_pg_pix_kernel<C, TW, TH, PG, MINB, true>
                       : warp_var_smem_pg_pix_kernel<C, TW, TH, PG, MINB, false>;
      if (form == kLadderInverse)
        return blocked ? warp_var_smem_pg_inv_kernel<C, TW, TH, PG, MINB, true>
                       : warp_var_smem_pg_inv_kernel<C, TW, TH, PG, MINB, false>;
      return blocked ? warp_var_smem_pg_kernel<C, TW, TH, PG, MINB, true>
                     : warp_var_smem_pg_kernel<C, TW, TH, PG, MINB, false>;
    } else {
      if (form == kLadderPixelStep)
        return blocked ? warp_var_smem_pix_kernel<NSRC, C, TW, TH, MINB, GWC, true>
                       : warp_var_smem_pix_kernel<NSRC, C, TW, TH, MINB, GWC, false>;
      if (form == kLadderInverse)
        return blocked ? warp_var_smem_inv_kernel<NSRC, C, TW, TH, MINB, GWC, true>
                       : warp_var_smem_inv_kernel<NSRC, C, TW, TH, MINB, GWC, false>;
      return blocked ? warp_var_smem_kernel<NSRC, C, TW, TH, MINB, GWC, true>
                     : warp_var_smem_kernel<NSRC, C, TW, TH, MINB, GWC, false>;
    }
  }();
  static std::atomic<bool> attr_set[3][2][kMaxDevices];
  if (int rc = opt_in_smem(kfn, 200 * 1024, attr_set[form][blocked ? 1 : 0], "warp_cost"))
    return rc;
  CUtensorMap map;
  if (int rc = feature_map(&map, feats, B * (NSRC + 1), h, w, C, BW, BH)) return rc;
  // depth runs: long enough to amortise the staging (a box is re-used by every plane of the
  // run), short enough to keep the sweep inside the margin and >= ~4 CTAs per SM in flight
  const int tiles_x = (w + TW - 1) / TW, tiles_y = (h + TH - 1) / TH;
  int dchunk = D <= 16 ? D : 16;
  while (dchunk > 4 && (long)tiles_x * tiles_y * B * ((D + dchunk - 1) / dchunk) < (long)num_sms() * 8)
    dchunk = (dchunk + 1) / 2;
  dim3 grd((unsigned)(tiles_x * tiles_y), (unsigned)B, (unsigned)((D + dchunk - 1) / dchunk));
  kfn<<<grd, NT, smem, st>>>(map, feats, proj, dv, cost, D, h, w, dchunk, BW, BH, box_stride,
                             tiles_x, rnd);
  return after_launch(PG > 0 ? "warp_cost(smem,pg)" : "warp_cost(smem)");
}

// Coverage: the shapes the staged kernels are instantiated for (V-1 source views, C channels,
// variance or 8-group correlation).  V-1 > 2 stays on the gather kernel: the staged boxes would
// leave one CTA per SM, and the gather kernel is faster there (cfg4 / cfg5).
// Variance, V-1 = 2: plane groups of 2, a view's window is re-used across the planes of a
// group.  Tried and removed: plane groups of 4 (spill at 128 registers), no window reuse (every
// plane loads its 2x2 windows; slower), windows of both views kept in registers across ALL
// planes (register pressure or spills through the same LSU pipe), coordinate math shared
// between the threads of a pixel by warp shuffles (shuffles use the bound pipe), 16 channels
// per thread (register pressure).
struct Shape {
  int nsrc, c, groups;
  StagedK1 run;
};
static const Shape kShapes[] = {
    {2, 8, 1, launch<2, 8, 32, 4, 4, false, 2>},  {2, 16, 1, launch<2, 16, 32, 2, 4, false, 2>},
    {2, 32, 1, launch<2, 32, 16, 2, 4, false, 2>},
    {1, 8, 1, launch<1, 8, 32, 4, 5, false, 0>},  {1, 16, 1, launch<1, 16, 32, 2, 5, false, 0>},
    {1, 32, 1, launch<1, 32, 16, 2, 5, false, 0>},
    // group-wise correlation: the reference's default G = 8
    {1, 8, 8, launch<1, 8, 32, 4, 5, true, 0>},   {1, 16, 8, launch<1, 16, 32, 2, 5, true, 0>},
    {1, 32, 8, launch<1, 32, 16, 2, 5, true, 0>},
    {2, 8, 8, launch<2, 8, 32, 4, 5, true, 0>},   {2, 16, 8, launch<2, 16, 32, 2, 5, true, 0>},
    {2, 32, 8, launch<2, 32, 16, 2, 5, true, 0>},
};

}  // namespace k1s

// CASMVS_K1_SMEM=0 leaves every shape to the gather kernel (the reference of the staged kernels).
StagedK1 warp_cost_staged(int V, int C, int num_groups) {
  if (!switches().k1_smem) return nullptr;
  for (const k1s::Shape& s : k1s::kShapes)
    if (s.nsrc == V - 1 && s.c == C && s.groups == num_groups) return s.run;
  return nullptr;
}

}  // namespace casmvs
