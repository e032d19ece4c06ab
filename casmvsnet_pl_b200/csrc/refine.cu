// Refine a mesh against its views: move each vertex along its normal to where its views agree
// (casmvsnet_pl_b200/refine.py drives these; oracle/refine_oracle.py restates them in float64).
//
// The rule, per iteration it = 0 .. T-1 (include/casmvs.h and the README state it too):
// 1. normals: n_v = the normalised sum, in double and in ascending face order, of the unnormalised
//    normals (x1 - x0) x (x2 - x0) of v's faces; a zero sum makes v unseen (n_v = 0);
// 2. visibility: v is visible in view j when it passes texture's step-2 vertex test against the
//    view's key buffer of the current mesh (w > 0, PAD <= u <= W-1-PAD, PAD <= v <= H-1-PAD,
//    w <= depth (1 + DEPTH_TOL) at the nearest pixel) and |cos(n_v, eye_j - v)| >= MIN_COS; one
//    bit per (vertex, view);
// 3. views: the reference is the visible view of largest |cos| (ties to the lower index); the
//    sources are the reference's pair-file sources in which v is visible, in pair order, at most
//    S_MAX; without a reference or a source v is unseen;
// 4. sweep: rho = the world distance between the back-projections through inv(P_ref) of v's pixel
//    (u, v) and (u + 1, v) at v's depth; t1 = normalise(a x n), a the axis of n's least |component|
//    (ties to the lower axis), t2 = n x t1; candidates k = -K .. K at delta_k = k rho STEP / 2^it;
//    patch points X = v + delta_k n + SPACING rho (a t1 + b t2), a, b = -R .. R.  Samples are bilinear in
//    the grey image g = (0.299 R + 0.587 G + 0.114 B) / 255, pixel centres at integer coordinates,
//    valid when w > 0 and all four taps lie inside.  A source counts for k when all its samples and
//    the reference's are valid and both population variances are >= VAR_MIN; S_k is the mean ZNCC
//    over the counting sources, and k is valid when one counts;
// 5. choice: k* = the valid k of largest S_k, ties to the smaller |k|, then the smaller k; when
//    k = 0 is valid and S_k* - S_0 < MIN_GAIN, k* = 0 instead; a parabolic sub-step
//    t = clamp((S- - S+) / (2 (S- - 2 S* + S+)), +-0.5) when k* != 0 is interior, both neighbours
//    are valid and the curvature is negative, else 0; d = (k* + t) step;
//    c = S* when k = 0 is valid and S* >= MIN_SCORE, else c = 0 and d = 0; unseen vertices
//    have c = 0;
// 6. regularise: J Jacobi rounds d <- (c d0 + lambda sum_{u in N(v)} d_u) / (c + lambda |N(v)|)
//    over the one-ring in ascending vertex order (0 for c = 0 without neighbours), then
//    v <- v + d n.
//
// Each vertex is one thread in every kernel and every sum has a fixed order; there are no atomics,
// so two runs give the same bits.  The sweep projects a patch point by linearity, q(X) = q(v) +
// delta q(n) + a SPACING rho q(t1) + b SPACING rho q(t2) with q the homogeneous projection, which differs from
// projecting X itself only by rounding.
#include <math_constants.h>

#include "render_common.cuh"

namespace casmvs {

constexpr int kRefR = 2;                      // patch half-width: (2R + 1)^2 = 25 points
constexpr int kRefK = 4;                      // candidates k = -K .. K
constexpr double kRefStep = 1.0;              // candidate spacing in footprints at it = 0
constexpr double kRefSpacing = 4.0;           // patch point spacing in footprints
constexpr double kRefMinGain = 5e-4;          // a move must beat S_0 by this much
constexpr int kRefSMax = 4;                   // sources per vertex
constexpr double kRefVarMin = 1e-4;
constexpr double kRefMinScore = 0.3;
constexpr double kRefLambda = 1.0;
constexpr int kRefPad = 2;                    // texture's PAD
constexpr double kRefMinCos = 0.1;            // texture's MIN_COS
constexpr float kRefDepthScale = 1.01f;       // 1 + texture's DEPTH_TOL
constexpr int kRefMaxBatch = 8;               // views per visibility call (texture's VIEW_BATCH)
constexpr int kRefMaxSide = 16384;
constexpr int kRefN = (2 * kRefR + 1) * (2 * kRefR + 1);
constexpr int kRefNK = 2 * kRefK + 1;
constexpr int kRefNoK = -1000;                // kstar of a vertex without a valid candidate

struct RefView {
  float P[12];
  double eye[3];
  const unsigned long long* zbuf;
  int W, H, index;
};
struct RefBatch {
  RefView v[kRefMaxBatch];
  int n;
};

__global__ void __launch_bounds__(256)
refine_grey_kernel(const unsigned char* __restrict__ rgb, long long n, double* __restrict__ grey) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double r = rgb[3 * i], g = rgb[3 * i + 1], b = rgb[3 * i + 2];
  grey[i] = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(0.299, r), __dmul_rn(0.587, g)),
                                __dmul_rn(0.114, b)), 255.0);
}

// Step 1: every operation rounded as written, so the oracle's numpy order gives the same bits.
__global__ void __launch_bounds__(256)
refine_normals_kernel(const float* __restrict__ verts, int V, const int* __restrict__ faces,
                      const int* __restrict__ vf_ptr, const int* __restrict__ vf_face,
                      double* __restrict__ normal) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  double s[3] = {0.0, 0.0, 0.0};
  for (int e = __ldg(vf_ptr + v), end = __ldg(vf_ptr + v + 1); e < end; ++e) {
    const int f = __ldg(vf_face + e);
    double x[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i = __ldg(faces + 3ll * f + k);
#pragma unroll
      for (int a = 0; a < 3; ++a) x[k][a] = (double)__ldg(verts + 3ll * i + a);
    }
    double e1[3], e2[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      e1[a] = __dsub_rn(x[1][a], x[0][a]);
      e2[a] = __dsub_rn(x[2][a], x[0][a]);
    }
    s[0] = __dadd_rn(s[0], __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1])));
    s[1] = __dadd_rn(s[1], __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2])));
    s[2] = __dadd_rn(s[2], __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0])));
  }
  const double nn = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(s[0], s[0]), __dmul_rn(s[1], s[1])),
                                         __dmul_rn(s[2], s[2])));
#pragma unroll
  for (int a = 0; a < 3; ++a) normal[3ll * v + a] = nn > 0.0 ? __ddiv_rn(s[a], nn) : 0.0;
}

// Step 2 for one batch of views: each thread read-modify-writes its own vertex's words only.
__global__ void __launch_bounds__(256)
refine_visibility_kernel(const __grid_constant__ RefBatch B, const float* __restrict__ verts,
                         const double* __restrict__ normal, int V, unsigned* __restrict__ vis,
                         int words) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const float x = __ldg(verts + 3ll * v), y = __ldg(verts + 3ll * v + 1), z = __ldg(verts + 3ll * v + 2);
  const double n[3] = {normal[3ll * v], normal[3ll * v + 1], normal[3ll * v + 2]};
  for (int b = 0; b < B.n; ++b) {
    const RefView& Vw = B.v[b];
    RenderCam cam;
#pragma unroll
    for (int r = 0; r < 12; ++r) cam.P[r] = Vw.P[r];
    float u, vv, w;
    if (!project(cam, x, y, z, u, vv, w)) continue;
    if (!(u >= (float)kRefPad && u <= (float)(Vw.W - 1 - kRefPad) && vv >= (float)kRefPad &&
          vv <= (float)(Vw.H - 1 - kRefPad)))
      continue;
    const unsigned long long key = Vw.zbuf[(size_t)(int)rintf(vv) * Vw.W + (int)rintf(u)];
    if (key == kKeyEmpty || !(w <= __fmul_rn(__uint_as_float((unsigned)(key >> 32)), kRefDepthScale)))
      continue;
    const double d[3] = {__dsub_rn(Vw.eye[0], (double)x), __dsub_rn(Vw.eye[1], (double)y),
                         __dsub_rn(Vw.eye[2], (double)z)};
    const double nd = __dadd_rn(__dadd_rn(__dmul_rn(n[0], d[0]), __dmul_rn(n[1], d[1])), __dmul_rn(n[2], d[2]));
    const double dd = __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]));
    if (!(fabs(nd) >= __dmul_rn(kRefMinCos, __dsqrt_rn(dd)))) continue;
    unsigned* word = vis + (size_t)v * words + (Vw.index >> 5);
    *word |= 1u << (Vw.index & 31);
  }
}

// Step 3.  src (V, S_MAX) int32, -1 past the last source; ref = -1 for an unseen vertex.
__global__ void __launch_bounds__(256)
refine_select_kernel(const float* __restrict__ verts, const double* __restrict__ normal, int V,
                     const unsigned* __restrict__ vis, int words, int n_views,
                     const double* __restrict__ eyes, const int* __restrict__ src_ptr,
                     const int* __restrict__ src_ids, int* __restrict__ ref, int* __restrict__ src) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const double x[3] = {(double)__ldg(verts + 3ll * v), (double)__ldg(verts + 3ll * v + 1),
                       (double)__ldg(verts + 3ll * v + 2)};
  const double n[3] = {normal[3ll * v], normal[3ll * v + 1], normal[3ll * v + 2]};
  const unsigned* bits = vis + (size_t)v * words;
  int best = -1;
  double best_cos = -1.0;
  for (int j = 0; j < n_views; ++j) {
    if (!((__ldg(bits + (j >> 5)) >> (j & 31)) & 1u)) continue;
    double d[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) d[a] = __dsub_rn(eyes[3 * j + a], x[a]);
    const double nd = __dadd_rn(__dadd_rn(__dmul_rn(n[0], d[0]), __dmul_rn(n[1], d[1])), __dmul_rn(n[2], d[2]));
    const double dd = __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]));
    const double c = __ddiv_rn(fabs(nd), __dsqrt_rn(dd));
    if (c > best_cos) { best_cos = c; best = j; }
  }
  int m = 0;
  if (best >= 0) {
    for (int e = __ldg(src_ptr + best), end = __ldg(src_ptr + best + 1); e < end && m < kRefSMax; ++e) {
      const int s = __ldg(src_ids + e);
      if ((__ldg(bits + (s >> 5)) >> (s & 31)) & 1u) src[(size_t)v * kRefSMax + m++] = s;
    }
  }
  ref[v] = m > 0 ? best : -1;
  for (int i = m; i < kRefSMax; ++i) src[(size_t)v * kRefSMax + i] = -1;
}

struct RefProj {
  double q0[3], qn[3], q1[3], q2[3];          // homogeneous q(v), q(n), rho q(t1), rho q(t2)
};

__device__ __forceinline__ void ref_proj(const float* P, const double x[3], const double n[3],
                                         const double t1[3], const double t2[3], double rho,
                                         RefProj& p) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double a0 = P[4 * r], a1 = P[4 * r + 1], a2 = P[4 * r + 2], a3 = P[4 * r + 3];
    p.q0[r] = a0 * x[0] + a1 * x[1] + a2 * x[2] + a3;
    p.qn[r] = a0 * n[0] + a1 * n[1] + a2 * n[2];
    p.q1[r] = rho * (a0 * t1[0] + a1 * t1[1] + a2 * t1[2]);
    p.q2[r] = rho * (a0 * t2[0] + a1 * t2[1] + a2 * t2[2]);
  }
}

// bilinear sample of the grey image at the patch point (a, b) of candidate delta; false when
// w <= 0 or a tap lies outside
__device__ __forceinline__ bool ref_sample(const RefProj& p, double delta, int a, int b,
                                           const double* __restrict__ g, int W, int H, double& out) {
  double q[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) q[r] = p.q0[r] + delta * p.qn[r] + (double)a * p.q1[r] + (double)b * p.q2[r];
  if (!(q[2] > 0.0)) return false;
  const double iw = 1.0 / q[2];
  const double u = q[0] * iw, v = q[1] * iw;
  if (!(u >= 0.0 && u < (double)(W - 1) && v >= 0.0 && v < (double)(H - 1))) return false;
  const double fx = floor(u), fy = floor(v);
  const double ax = u - fx, ay = v - fy;
  const double* r0 = g + (size_t)(int)fy * W + (int)fx;
  const double* r1 = r0 + W;
  const double c0 = (1.0 - ax) * __ldg(r0) + ax * __ldg(r0 + 1);
  const double c1 = (1.0 - ax) * __ldg(r1) + ax * __ldg(r1 + 1);
  out = (1.0 - ay) * c0 + ay * c1;
  return true;
}

// Steps 4-5, the hot path.  sk (V, 2K+1) f64, NaN for an invalid k, is written only when given.
__global__ void __launch_bounds__(128)
refine_sweep_kernel(const float* __restrict__ verts, const double* __restrict__ normal, int V,
                    const int* __restrict__ ref, const int* __restrict__ src,
                    const float* __restrict__ Ps, const double* __restrict__ Pinv,
                    const unsigned long long* __restrict__ grey, const int* __restrict__ wh,
                    double scale, double* __restrict__ rho_out, double* __restrict__ best_out,
                    int* __restrict__ kstar_out, double* __restrict__ d_out,
                    double* __restrict__ conf_out, double* __restrict__ sk_out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int r = __ldg(ref + v);
  double rho = 0.0, best = CUDART_NAN, d = 0.0, conf = 0.0;
  int kstar = kRefNoK;
  double sk[kRefNK];
#pragma unroll
  for (int i = 0; i < kRefNK; ++i) sk[i] = CUDART_NAN;
  if (r >= 0) {
    const double x[3] = {(double)__ldg(verts + 3ll * v), (double)__ldg(verts + 3ll * v + 1),
                         (double)__ldg(verts + 3ll * v + 2)};
    const double n[3] = {normal[3ll * v], normal[3ll * v + 1], normal[3ll * v + 2]};
    // rho: the footprint of v's pixel at v's depth in the reference view
    const float* Pr = Ps + (size_t)r * 16;
    double qz = 0.0, qu = 0.0, qv = 0.0;
    {
      double q[3];
#pragma unroll
      for (int i = 0; i < 3; ++i)
        q[i] = (double)Pr[4 * i] * x[0] + (double)Pr[4 * i + 1] * x[1] + (double)Pr[4 * i + 2] * x[2] +
               (double)Pr[4 * i + 3];
      qz = q[2];
      qu = q[0] / qz;
      qv = q[1] / qz;
    }
    const double* Mi = Pinv + (size_t)r * 16;
    double A[4], Bv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const double base = Mi[4 * i + 1] * (qv * qz) + Mi[4 * i + 2] * qz + Mi[4 * i + 3];
      A[i] = Mi[4 * i] * (qu * qz) + base;
      Bv[i] = Mi[4 * i] * ((qu + 1.0) * qz) + base;
    }
    double rr = 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const double e = A[i] / A[3] - Bv[i] / Bv[3];
      rr += e * e;
    }
    rho = sqrt(rr);
    if (qz > 0.0 && rho > 0.0 && isfinite(rho)) {
      // tangent frame
      int ax = 0;
      if (fabs(n[1]) < fabs(n[ax])) ax = 1;
      if (fabs(n[2]) < fabs(n[ax])) ax = 2;
      double c[3];                              // e_ax x n
      c[0] = ax == 1 ? n[2] : (ax == 2 ? -n[1] : 0.0);
      c[1] = ax == 2 ? n[0] : (ax == 0 ? -n[2] : 0.0);
      c[2] = ax == 0 ? n[1] : (ax == 1 ? -n[0] : 0.0);
      const double cl = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
      const double t1[3] = {c[0] / cl, c[1] / cl, c[2] / cl};
      const double t2[3] = {n[1] * t1[2] - n[2] * t1[1], n[2] * t1[0] - n[0] * t1[2],
                            n[0] * t1[1] - n[1] * t1[0]};
      const double step = rho * kRefStep * scale;
      RefProj pr;
      ref_proj(Pr, x, n, t1, t2, rho * kRefSpacing, pr);
      const double* gr = reinterpret_cast<const double*>(grey[r]);
      const int Wr = wh[2 * r], Hr = wh[2 * r + 1];
      int ns = 0, sid[kRefSMax];
#pragma unroll
      for (int i = 0; i < kRefSMax; ++i) {
        sid[i] = __ldg(src + (size_t)v * kRefSMax + i);
        if (sid[i] >= 0) ns = i + 1;
      }
      for (int k = -kRefK; k <= kRefK; ++k) {
        const double delta = (double)k * step;
        double g[kRefN];
        bool ok = true;
        double sx = 0.0;
#pragma unroll
        for (int b = -kRefR; b <= kRefR; ++b)
#pragma unroll
          for (int a = -kRefR; a <= kRefR; ++a) {
            double s = 0.0;
            ok = ok && ref_sample(pr, delta, a, b, gr, Wr, Hr, s);
            g[(b + kRefR) * (2 * kRefR + 1) + a + kRefR] = s;
            sx += s;
          }
        if (!ok) continue;
        const double mx = sx / kRefN;
        double vx = 0.0;
#pragma unroll
        for (int i = 0; i < kRefN; ++i) {
          g[i] -= mx;
          vx += g[i] * g[i];
        }
        vx /= kRefN;
        if (!(vx >= kRefVarMin)) continue;
        double zsum = 0.0;
        int cnt = 0;
        for (int s = 0; s < ns; ++s) {
          const int j = sid[s];
          RefProj ps;
          ref_proj(Ps + (size_t)j * 16, x, n, t1, t2, rho * kRefSpacing, ps);
          const double* gs = reinterpret_cast<const double*>(grey[j]);
          const int Ws = wh[2 * j], Hs = wh[2 * j + 1];
          double sy = 0.0, syy = 0.0, sxy = 0.0;
          bool oks = true;
#pragma unroll
          for (int b = -kRefR; b <= kRefR; ++b)
#pragma unroll
            for (int a = -kRefR; a <= kRefR; ++a) {
              double y = 0.0;
              oks = oks && ref_sample(ps, delta, a, b, gs, Ws, Hs, y);
              y -= mx;
              sy += y;
              syy += y * y;
              sxy += g[(b + kRefR) * (2 * kRefR + 1) + a + kRefR] * y;
            }
          if (!oks) continue;
          const double my = sy / kRefN;
          const double vy = syy / kRefN - my * my;
          if (!(vy >= kRefVarMin)) continue;
          zsum += (sxy / kRefN) / sqrt(vx * vy);
          ++cnt;
        }
        if (cnt > 0) sk[k + kRefK] = zsum / cnt;
      }
      // k* over the order 0, -1, +1, -2, +2, ...: a strictly larger score wins, so ties go to the
      // smaller |k|, then the smaller k
#pragma unroll
      for (int m = 0; m <= 2 * kRefK; ++m) {
        const int k = (m & 1) ? -((m + 1) >> 1) : (m >> 1);
        const double s = sk[k + kRefK];
        if (s == s && (kstar == kRefNoK || s > best)) { best = s; kstar = k; }
      }
      // a valid k = 0 stays unless k* beats it by MIN_GAIN
      if (kstar != kRefNoK && sk[kRefK] == sk[kRefK] && best - sk[kRefK] < kRefMinGain) {
        kstar = 0;
        best = sk[kRefK];
      }
      if (kstar != kRefNoK) {
        double t = 0.0;
        if (kstar != 0 && kstar > -kRefK && kstar < kRefK) {
          const double sm = sk[kstar + kRefK - 1], sp = sk[kstar + kRefK + 1];
          const double curv = sm - 2.0 * best + sp;
          if (sm == sm && sp == sp && curv < 0.0) t = fmin(fmax((sm - sp) / (2.0 * curv), -0.5), 0.5);
        }
        if (sk[kRefK] == sk[kRefK] && best >= kRefMinScore) {
          conf = best;
          d = ((double)kstar + t) * step;
        }
      }
    }
  }
  rho_out[v] = rho;
  best_out[v] = best;
  kstar_out[v] = kstar;
  d_out[v] = d;
  conf_out[v] = conf;
  if (sk_out) {
#pragma unroll
    for (int i = 0; i < kRefNK; ++i) sk_out[(size_t)v * kRefNK + i] = sk[i];
  }
}

// Step 6: one Jacobi round.
__global__ void __launch_bounds__(256)
refine_smooth_kernel(const int* __restrict__ nb_ptr, const int* __restrict__ nb_ids, int V,
                     const double* __restrict__ d0, const double* __restrict__ conf,
                     const double* __restrict__ din, double* __restrict__ dout) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int b = __ldg(nb_ptr + v), e = __ldg(nb_ptr + v + 1);
  double s = 0.0;
  for (int i = b; i < e; ++i) s += din[__ldg(nb_ids + i)];
  const double c = conf[v];
  const double den = c + kRefLambda * (double)(e - b);
  dout[v] = den > 0.0 ? (c * d0[v] + kRefLambda * s) / den : 0.0;
}

__global__ void __launch_bounds__(256)
refine_apply_kernel(const float* __restrict__ vin, const double* __restrict__ normal,
                    const double* __restrict__ d, int V, float* __restrict__ vout) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3ll * V) return;
  vout[i] = __double2float_rn(__dadd_rn((double)vin[i], __dmul_rn(d[i / 3], normal[i])));
}

inline unsigned ref_blocks(long long n, int t = 256) { return (unsigned)((n + t - 1) / t); }

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_refine_grey(const unsigned char* rgb, long long n_pixels, double* grey,
                                  void* stream) {
  const char* what = "refine_grey";
  CASMVS_REQUIRE(n_pixels >= 0, "%s: n_pixels < 0", what);
  if (n_pixels == 0) return 0;
  CASMVS_REQUIRE(rgb && grey, "%s: null pointer", what);
  refine_grey_kernel<<<ref_blocks(n_pixels), 256, 0, as_stream(stream)>>>(rgb, n_pixels, grey);
  return after_launch(what);
}

extern "C" int casmvs_refine_normals(const float* verts, int V, const int* faces, const int* vf_ptr,
                                     const int* vf_face, double* normal, void* stream) {
  const char* what = "refine_normals";
  CASMVS_REQUIRE(V >= 0, "%s: V < 0", what);
  if (V == 0) return 0;
  CASMVS_REQUIRE(verts && vf_ptr && normal, "%s: null pointer", what);
  refine_normals_kernel<<<ref_blocks(V), 256, 0, as_stream(stream)>>>(verts, V, faces, vf_ptr, vf_face,
                                                                      normal);
  return after_launch(what);
}

extern "C" int casmvs_refine_visibility(const float* verts, const double* normal, int V, int n_views,
                                        const float* P, const double* eye, const int* wh,
                                        const int* view_index, unsigned long long* const* zbufs,
                                        unsigned* vis, int words, void* stream) {
  const char* what = "refine_visibility";
  CASMVS_REQUIRE(V >= 0 && n_views >= 0 && n_views <= kRefMaxBatch && words >= 0,
                 "%s: need V >= 0, 0 <= n_views <= %d and words >= 0 (got %d, %d, %d)", what,
                 kRefMaxBatch, V, n_views, words);
  if (V == 0 || n_views == 0) return 0;
  CASMVS_REQUIRE(verts && normal && P && eye && wh && view_index && zbufs && vis, "%s: null pointer",
                 what);
  RefBatch B;
  B.n = n_views;
  for (int j = 0; j < n_views; ++j) {
    for (int r = 0; r < 12; ++r) B.v[j].P[r] = P[j * 16 + r];
    for (int a = 0; a < 3; ++a) B.v[j].eye[a] = eye[j * 3 + a];
    B.v[j].W = wh[2 * j];
    B.v[j].H = wh[2 * j + 1];
    B.v[j].index = view_index[j];
    B.v[j].zbuf = zbufs[j];
    CASMVS_REQUIRE(B.v[j].W > 2 * kRefPad && B.v[j].H > 2 * kRefPad && B.v[j].W <= kRefMaxSide &&
                   B.v[j].H <= kRefMaxSide && zbufs[j] && view_index[j] >= 0 &&
                   (view_index[j] >> 5) < words, "%s: view %d: bad size %d x %d, index or null key "
                   "buffer", what, view_index[j], B.v[j].W, B.v[j].H);
  }
  refine_visibility_kernel<<<ref_blocks(V), 256, 0, as_stream(stream)>>>(B, verts, normal, V, vis, words);
  return after_launch(what);
}

extern "C" int casmvs_refine_select(const float* verts, const double* normal, int V,
                                    const unsigned* vis, int words, int n_views, const double* eyes,
                                    const int* src_ptr, const int* src_ids, int* ref, int* src,
                                    void* stream) {
  const char* what = "refine_select";
  CASMVS_REQUIRE(V >= 0 && n_views >= 0 && words * 32 >= n_views, "%s: need V >= 0, n_views >= 0 "
                 "and 32 words >= n_views (got %d, %d, %d)", what, V, n_views, words);
  if (V == 0) return 0;
  CASMVS_REQUIRE(verts && normal && ref && src && (n_views == 0 || (vis && eyes && src_ptr)),
                 "%s: null pointer", what);
  refine_select_kernel<<<ref_blocks(V), 256, 0, as_stream(stream)>>>(verts, normal, V, vis, words, n_views,
                                                                     eyes, src_ptr, src_ids, ref, src);
  return after_launch(what);
}

extern "C" int casmvs_refine_sweep(const float* verts, const double* normal, int V, const int* ref,
                                   const int* src, const float* Ps, const double* Pinv,
                                   const unsigned long long* grey, const int* wh, int iteration,
                                   double* rho, double* best, int* kstar, double* d, double* conf,
                                   double* sk, void* stream) {
  const char* what = "refine_sweep";
  CASMVS_REQUIRE(V >= 0 && iteration >= 0 && iteration < 64, "%s: need V >= 0 and 0 <= iteration "
                 "< 64 (got %d, %d)", what, V, iteration);
  if (V == 0) return 0;
  CASMVS_REQUIRE(verts && normal && ref && src && Ps && Pinv && grey && wh && rho && best && kstar &&
                 d && conf, "%s: null pointer", what);
  refine_sweep_kernel<<<ref_blocks(V, 128), 128, 0, as_stream(stream)>>>(
      verts, normal, V, ref, src, Ps, Pinv, grey, wh, ldexp(1.0, -iteration), rho, best, kstar, d,
      conf, sk);
  return after_launch(what);
}

extern "C" int casmvs_refine_smooth(const int* nb_ptr, const int* nb_ids, int V, const double* d0,
                                    const double* conf, const double* d_in, double* d_out,
                                    void* stream) {
  const char* what = "refine_smooth";
  CASMVS_REQUIRE(V >= 0, "%s: V < 0", what);
  if (V == 0) return 0;
  CASMVS_REQUIRE(nb_ptr && d0 && conf && d_in && d_out && d_in != d_out, "%s: null or aliased pointer",
                 what);
  refine_smooth_kernel<<<ref_blocks(V), 256, 0, as_stream(stream)>>>(nb_ptr, nb_ids, V, d0, conf, d_in,
                                                                     d_out);
  return after_launch(what);
}

extern "C" int casmvs_refine_apply(const float* verts_in, const double* normal, const double* d,
                                   int V, float* verts_out, void* stream) {
  const char* what = "refine_apply";
  CASMVS_REQUIRE(V >= 0, "%s: V < 0", what);
  if (V == 0) return 0;
  CASMVS_REQUIRE(verts_in && normal && d && verts_out, "%s: null pointer", what);
  refine_apply_kernel<<<ref_blocks(3ll * V), 256, 0, as_stream(stream)>>>(verts_in, normal, d, V,
                                                                          verts_out);
  return after_launch(what);
}
