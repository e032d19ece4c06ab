// Geometric-consistency filter + depth / colour refinement + back-projection on the GPU
// (SURVEY.md 8 f-3): the consumer of depth_0 / confidence_2 right after the hot path.
//
// Replaces (reference, paths relative to /root/reference):
//   xy_ref2src, xy_src2ref, check_geo_consistency       eval.py:113-182  (numba + cv2.remap, CPU)
//   mask / average / back-projection of one ref view    eval.py:262-318
// One thread per reference pixel walks the source views: project with the reference depth,
// sample the source depth map and image bilinearly (cv2.remap semantics, see remap_tap), lift
// back, measure e_pix = dx^2 + dy^2 and e_dep = |(rz - d) / d|, accumulate.  Two rules decide
// from those errors, one template instantiation each (FuseRule):
//   reference  a source is consistent when e_pix < 1 and e_dep < 0.01f; the pixel passes when
//              at least min_consistent sources are (eval.py:143-147,300).
//   dynamic    dynamic consistency checking (D2HC-RMVSNet, Yan et al., ECCV 2020, in its
//              count-based form).  Source s is consistent at level k (k = 2..10) when
//              e_pix < (k/4)^2 and e_dep < T_k = float32(k / 1300) (rounded once from double);
//              k_s is its least such level, 0 when there is none (NaN compares false).  With
//              n_k = #{s : 0 < k_s <= k}, the pixel passes when n_k >= k for some
//              2 <= k <= min(10, S); with S < 2 it never does.  The average and geo_count use
//              the sources with k_s > 0 (consistent at level 10).
// Both then AND the confidence test.  HBM-bound, the same bytes for both rules: per ref pixel
// it reads 4 B + S x (4 taps x 16 B) and writes 4 + 12 + 4 (+ 12 + 1) bytes; the depth
// maps of a scan stay resident, so the PFM round trip of eval.py:228-229,269-272 disappears.
#include "common.cuh"

namespace casmvs {

constexpr int kMaxFuseSrc = 16;

// The dynamic rule's constants (fusion.py states them again; a test keeps the two in step):
// levels k = kDynLevelMin..kDynLevelMax, pixel threshold k / kDynPixDiv px, relative depth
// threshold k / kDynDepDiv.
constexpr int kDynLevelMin = 2;
constexpr int kDynLevelMax = 10;
constexpr int kDynPixDiv = 4;
constexpr int kDynDepDiv = 1300;
// geo_fuse_kernel<kDynamic> counts the sources per level in 5-bit fields of one 64-bit word
constexpr int kDynCountBits = 5;
static_assert(kMaxFuseSrc < (1 << kDynCountBits), "a level count must fit its field");
static_assert((kDynLevelMax - kDynLevelMin + 1) * kDynCountBits <= 64, "level counts overflow");

enum class FuseRule { kReference, kDynamic };

struct FuseParams {
  float rs[kMaxFuseSrc][12];   // (P_world2src @ inv(P_world2ref))[:3]   eval.py:120
  float sr[kMaxFuseSrc][12];   // (P_world2ref @ inv(P_world2src))[:3]   eval.py:136
  const float* depth_src[kMaxFuseSrc];
  const float* image_src[kMaxFuseSrc];
};

// cv2.remap(INTER_LINEAR, BORDER_CONSTANT 0) with float32 maps: coordinates are rounded to
// 1/32 px (INTER_BITS = 5, cvRound = round-half-even), weights come from the exact table
// (1-fx)(1-fy), fx(1-fy), (1-fx)fy, fx*fy and out-of-image taps read the border value 0.
struct RemapPos { int ix, iy; float w00, w01, w10, w11; };
__device__ __forceinline__ RemapPos remap_pos(float x, float y) {
  // __float2int_rn saturates and maps NaN to 0; cv2 maps NaN to INT_MIN (outside): handled by
  // the caller's finite test
  const int sx = __float2int_rn(x * 32.f), sy = __float2int_rn(y * 32.f);
  RemapPos p;
  p.ix = sx >> 5; p.iy = sy >> 5;
  const float fx = (float)(sx & 31) * (1.f / 32.f), fy = (float)(sy & 31) * (1.f / 32.f);
  p.w00 = (1.f - fx) * (1.f - fy); p.w01 = fx * (1.f - fy);
  p.w10 = (1.f - fx) * fy;         p.w11 = fx * fy;
  return p;
}

template <int NCH>
__device__ __forceinline__ void remap_sample(const float* __restrict__ img, int H, int W,
                                             const RemapPos& p, float (&out)[NCH]) {
  const bool x0 = (unsigned)p.ix < (unsigned)W, x1 = (unsigned)(p.ix + 1) < (unsigned)W;
  const bool y0 = (unsigned)p.iy < (unsigned)H, y1 = (unsigned)(p.iy + 1) < (unsigned)H;
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const float a = (x0 && y0) ? __ldg(img + ((size_t)p.iy * W + p.ix) * NCH + c) : 0.f;
    const float b = (x1 && y0) ? __ldg(img + ((size_t)p.iy * W + p.ix + 1) * NCH + c) : 0.f;
    const float d = (x0 && y1) ? __ldg(img + ((size_t)(p.iy + 1) * W + p.ix) * NCH + c) : 0.f;
    const float e = (x1 && y1) ? __ldg(img + ((size_t)(p.iy + 1) * W + p.ix + 1) * NCH + c) : 0.f;
    // remapBilinear: S0[0]*w[0] + S0[1]*w[1] + S1[0]*w[2] + S1[1]*w[3], left to right
    out[c] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, p.w00), __fmul_rn(b, p.w01)),
                                 __fmul_rn(d, p.w10)), __fmul_rn(e, p.w11));
  }
}

// cv2.resize(proba, fx=4, fy=4, INTER_LINEAR) at full-resolution pixel (x, y): source
// coordinate (dst + 0.5)/4 - 0.5, replicated border   (eval.py:273-275)
__device__ __forceinline__ float upsample4_linear(const float* __restrict__ p, int h4, int w4,
                                                  int x, int y) {
  float fx = (float)(((double)x + 0.5) * 0.25 - 0.5), fy = (float)(((double)y + 0.5) * 0.25 - 0.5);
  int sx = (int)floorf(fx), sy = (int)floorf(fy);
  fx -= (float)sx; fy -= (float)sy;
  if (sx < 0) { fx = 0.f; sx = 0; }
  if (sx >= w4 - 1) { fx = 0.f; sx = w4 - 1; }
  if (sy < 0) { fy = 0.f; sy = 0; }
  if (sy >= h4 - 1) { fy = 0.f; sy = h4 - 1; }
  const int sx1 = min(sx + 1, w4 - 1), sy1 = min(sy + 1, h4 - 1);
  const float r0 = __fadd_rn(__fmul_rn(__ldg(p + sy * w4 + sx), 1.f - fx),
                             __fmul_rn(__ldg(p + sy * w4 + sx1), fx));
  const float r1 = __fadd_rn(__fmul_rn(__ldg(p + sy1 * w4 + sx), 1.f - fx),
                             __fmul_rn(__ldg(p + sy1 * w4 + sx1), fx));
  return __fadd_rn(__fmul_rn(r0, 1.f - fy), __fmul_rn(r1, fy));
}

// Least level k at which a source with errors (e_pix, e_dep) is consistent, 0 for none.
// (k / kDynPixDiv)^2 = k^2 / 16 is exact in fp32, so the squared pixel error is compared.
__device__ __forceinline__ int dynamic_level(float e_pix, float e_dep) {
#pragma unroll
  for (int k = kDynLevelMin; k <= kDynLevelMax; ++k) {
    const float pix_th = (float)(k * k) / (float)(kDynPixDiv * kDynPixDiv);
    const float dep_th = (float)((double)k / (double)kDynDepDiv);
    if (e_pix < pix_th && e_dep < dep_th) return k;
  }
  return 0;
}

// R = kReference: flag_dbg holds the per-source mask (0 / 1) and min_consistent applies.
// R = kDynamic:   flag_dbg holds k_s and min_consistent is unused.
template <FuseRule R>
__global__ void __launch_bounds__(256)
geo_fuse_kernel(const __grid_constant__ FuseParams P, int S, const float* __restrict__ depth_ref,
                const float* __restrict__ image_ref, const float* __restrict__ proba_ref,
                float conf_thresh, int min_consistent, const float* __restrict__ ref2world,
                float* __restrict__ depth_refined, float* __restrict__ image_refined,
                int* __restrict__ geo_count, unsigned char* __restrict__ mask_final,
                float* __restrict__ points, float* __restrict__ reproj_dbg,
                unsigned char* __restrict__ flag_dbg, int H, int W) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= H * W) return;
  const int y = pix / W, x = pix - y * W;
  const float xf = (float)x, yf = (float)y;
  const float d = __ldg(depth_ref + pix);
  float dsum = d;                                      // depth_ref_reprojs = [depth_ref, ...]
  float csum[3] = {0.f, 0.f, 0.f};
  if (image_ref) {
#pragma unroll
    for (int c = 0; c < 3; ++c) csum[c] = __ldg(image_ref + (size_t)pix * 3 + c);
  }
  int cnt = 0;
  unsigned long long level_count = 0;   // kDynamic: sources per level, kDynCountBits each
  for (int s = 0; s < S; ++s) {
    const float* A = P.rs[s];
    // xyz_ref = (x, y, 1) * depth_ref; homogeneous 1      eval.py:117-118
    const float X = xf * d, Y = yf * d;
    const float qx = A[0] * X + A[1] * Y + A[2] * d + A[3];
    const float qy = A[4] * X + A[5] * Y + A[6] * d + A[7];
    const float qz = A[8] * X + A[9] * Y + A[10] * d + A[11];
    const float xs = qx / qz, ys = qy / qz;            // eval.py:123
    float ds = 0.f, col[3] = {0.f, 0.f, 0.f};
    if (isfinite(xs) && isfinite(ys)) {
      const RemapPos rp = remap_pos(xs, ys);
      float t[1];
      remap_sample<1>(P.depth_src[s], H, W, rp, t);    // eval.py:160-163
      ds = t[0];
      if (P.image_src[s]) remap_sample<3>(P.image_src[s], H, W, rp, col);   // :165-168
    }
    const float* Bm = P.sr[s];
    const float U = xs * ds, Vv = ys * ds;             // eval.py:134-135
    const float rx = Bm[0] * U + Bm[1] * Vv + Bm[2] * ds + Bm[3];
    const float ry = Bm[4] * U + Bm[5] * Vv + Bm[6] * ds + Bm[7];
    const float rz = Bm[8] * U + Bm[9] * Vv + Bm[10] * ds + Bm[11];
    const float dx = rx / rz - xf, dy = ry / rz - yf;
    bool m;                                            // the source joins the average
    unsigned char flag;
    if constexpr (R == FuseRule::kReference) {
      const bool m_pix = dx * dx + dy * dy < 1.f;                       // eval.py:143-144
      const bool m_dep = fabsf((rz - d) / d) < 0.01f;                   // eval.py:147
      m = m_pix && m_dep;                                               // NaN compares false
      flag = m ? 1 : 0;
    } else {
      const int level = dynamic_level(dx * dx + dy * dy, fabsf((rz - d) / d));
      m = level > 0;
      if (m) level_count += 1ull << (kDynCountBits * (level - kDynLevelMin));
      flag = (unsigned char)level;
    }
    if (m) {
      dsum += rz;                                      // depth_ref_reproj[~mask_geo] = 0
      csum[0] += col[0]; csum[1] += col[1]; csum[2] += col[2];
      ++cnt;
    }
    if (reproj_dbg) reproj_dbg[(size_t)s * H * W + pix] = m ? rz : 0.f;
    if (flag_dbg) flag_dbg[(size_t)s * H * W + pix] = flag;
  }
  const float inv = 1.f / (float)(cnt + 1);
  const float dref = dsum / (float)(cnt + 1);                            // eval.py:301-302
  depth_refined[pix] = dref;
  if (image_refined) {
#pragma unroll
    for (int c = 0; c < 3; ++c) image_refined[(size_t)pix * 3 + c] = csum[c] * inv;
  }
  geo_count[pix] = cnt;
  bool keep;
  if constexpr (R == FuseRule::kReference) {
    keep = cnt >= min_consistent;                                        // eval.py:300
  } else {
    keep = false;
    int n = 0;                                         // n_k = #{s : 0 < k_s <= k}
#pragma unroll
    for (int k = kDynLevelMin; k <= kDynLevelMax; ++k) {
      n += (int)((level_count >> (kDynCountBits * (k - kDynLevelMin))) & ((1u << kDynCountBits) - 1));
      keep = keep || (k <= S && n >= k);
    }
  }
  if (proba_ref) keep = keep && upsample4_linear(proba_ref, H / 4, W / 4, x, y) > conf_thresh;
  if (mask_final) mask_final[pix] = keep ? 1 : 0;
  if (points) {
    // xyz_world = inv(P_world2ref) @ (x*d, y*d, d, 1)      eval.py:311-315
    const float X = xf * dref, Y = yf * dref;
    const float* M = ref2world;
#pragma unroll
    for (int r = 0; r < 3; ++r)
      points[(size_t)pix * 3 + r] = __ldg(M + 4 * r) * X + __ldg(M + 4 * r + 1) * Y +
                                    __ldg(M + 4 * r + 2) * dref + __ldg(M + 4 * r + 3);
  }
}

}  // namespace casmvs

using namespace casmvs;

// Argument checks and launch shared by both entries.
template <FuseRule R>
static int geo_fuse_launch(const float* depth_ref, const float* image_ref, const float* proba_ref,
                           const float* const* depth_src, const float* const* image_src,
                           const float* proj_ref2src, const float* proj_src2ref,
                           const float* ref2world, int S, int H, int W, float conf_thresh,
                           int min_consistent, float* depth_refined, float* image_refined,
                           int* geo_count, unsigned char* mask_final, float* points,
                           float* reproj_dbg, unsigned char* flag_dbg, void* stream) {
  CASMVS_REQUIRE(depth_ref && depth_refined && geo_count, "geo_fuse: null pointer");
  CASMVS_REQUIRE(S >= 0 && S <= kMaxFuseSrc, "geo_fuse: at most %d source views", kMaxFuseSrc);
  CASMVS_REQUIRE(H > 0 && W > 0 && (size_t)H * W < (1u << 30), "geo_fuse: bad dims");
  CASMVS_REQUIRE(S == 0 || (depth_src && proj_ref2src && proj_src2ref), "geo_fuse: null sources");
  CASMVS_REQUIRE(!proba_ref || (H % 4 == 0 && W % 4 == 0), "geo_fuse: proba needs H,W %% 4 == 0");
  CASMVS_REQUIRE(!points || ref2world, "geo_fuse: points need ref2world");
  CASMVS_REQUIRE(!image_refined || image_ref, "geo_fuse: image_refined needs image_ref");
  FuseParams P;
  for (int s = 0; s < S; ++s) {
    CASMVS_REQUIRE(depth_src[s], "geo_fuse: null source depth %d", s);
    for (int k = 0; k < 12; ++k) {
      P.rs[s][k] = proj_ref2src[s * 12 + k];
      P.sr[s][k] = proj_src2ref[s * 12 + k];
    }
    P.depth_src[s] = depth_src[s];
    P.image_src[s] = (image_src && image_ref) ? image_src[s] : nullptr;
    CASMVS_REQUIRE(!image_ref || !image_src || image_src[s], "geo_fuse: null source image %d", s);
  }
  const int n = H * W;
  geo_fuse_kernel<R><<<(n + 255) / 256, 256, 0, as_stream(stream)>>>(
      P, S, depth_ref, image_ref, proba_ref, conf_thresh, min_consistent, ref2world, depth_refined,
      image_refined, geo_count, mask_final, points, reproj_dbg, flag_dbg, H, W);
  return after_launch("geo_fuse");
}

extern "C" int casmvs_geo_fuse_fwd(const float* depth_ref, const float* image_ref,
                                   const float* proba_ref, const float* const* depth_src,
                                   const float* const* image_src, const float* proj_ref2src,
                                   const float* proj_src2ref, const float* ref2world, int S, int H,
                                   int W, float conf_thresh, int min_consistent,
                                   float* depth_refined, float* image_refined, int* geo_count,
                                   unsigned char* mask_final, float* points, float* reproj_dbg,
                                   unsigned char* mask_dbg, void* stream) {
  return geo_fuse_launch<FuseRule::kReference>(
      depth_ref, image_ref, proba_ref, depth_src, image_src, proj_ref2src, proj_src2ref,
      ref2world, S, H, W, conf_thresh, min_consistent, depth_refined, image_refined, geo_count,
      mask_final, points, reproj_dbg, mask_dbg, stream);
}

extern "C" int casmvs_geo_fuse_dynamic_fwd(const float* depth_ref, const float* image_ref,
                                           const float* proba_ref, const float* const* depth_src,
                                           const float* const* image_src,
                                           const float* proj_ref2src, const float* proj_src2ref,
                                           const float* ref2world, int S, int H, int W,
                                           float conf_thresh, float* depth_refined,
                                           float* image_refined, int* geo_count,
                                           unsigned char* mask_final, float* points,
                                           float* reproj_dbg, unsigned char* level_dbg,
                                           void* stream) {
  return geo_fuse_launch<FuseRule::kDynamic>(
      depth_ref, image_ref, proba_ref, depth_src, image_src, proj_ref2src, proj_src2ref,
      ref2world, S, H, W, conf_thresh, 0, depth_refined, image_refined, geo_count, mask_final,
      points, reproj_dbg, level_dbg, stream);
}
