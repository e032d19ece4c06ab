// Level the colour seams of a textured mesh (Waechter et al. 2014, global adjustment): the seam
// edges and the per-(chart, vertex) unknowns, the seam colours sampled from the two views, the CSR
// system, Jacobi-preconditioned conjugate gradients over three right-hand sides, and the texel
// owners and the offsets applied to the atlas (casmvsnet_pl_b200/texture.py drives these;
// oracle/texture_level_oracle.py restates every step but the solve in numpy, bit for bit).
// include/casmvs.h states the rule.
//
// Every double operation the oracle restates is explicitly rounded (no contraction); each sum runs
// in one thread in a fixed order, and the CG's dot products are fixed-shape block trees over a
// grid whose size depends on n alone.  The only atomics are the 64-bit integer atomicMin of the
// owner pass, whose result does not depend on the schedule.
#include "render_common.cuh"

namespace casmvs {

constexpr int kLvSamples = 8;                 // SEAM_SAMPLES
constexpr double kLvSmooth = 10.0;            // SMOOTH_WEIGHT
constexpr double kLvEps = 1e-4;               // EPS
constexpr double kLvReach = 1.5;              // REACH, in texels
constexpr int kLvMaxSide = 16384;
constexpr int kLvThreads = 256;
constexpr int kLvMaxBlocks = 1024;            // CG reduction blocks

__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ long long lv_pair(int a, int b) {
  return ((long long)min(a, b) << 32) | (long long)max(a, b);
}

// ---------------------------------------------------------------- unknowns and seams
__global__ void __launch_bounds__(256)
level_keys_kernel(const int* __restrict__ faces, int F, const int* __restrict__ label,
                  const int* __restrict__ slot, long long* __restrict__ keys) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3ll * F) return;
  const int f = (int)(i / 3);
  keys[i] = __ldg(label + f) >= 0 ? ((long long)__ldg(slot + f) << 32) | (long long)__ldg(faces + i)
                                  : -1ll;
}

__global__ void __launch_bounds__(256)
level_corners_kernel(const long long* __restrict__ keys, int F, const long long* __restrict__ unk,
                     int n, int* __restrict__ corner) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3ll * F) return;
  const long long k = keys[i];
  if (k < 0) { corner[i] = -1; return; }
  int lo = 0, hi = n;                          // lower bound; k is present
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (unk[mid] < k) lo = mid + 1; else hi = mid;
  }
  corner[i] = lo;
}

// per corner (f, k): the smoothing edge of f's chart, and the two endpoint records of a seam edge
// seen from its lower face
__global__ void __launch_bounds__(256)
level_edges_kernel(const int* __restrict__ nbr, const int* __restrict__ faces, int F,
                   const int* __restrict__ label, const int* __restrict__ slot,
                   const int* __restrict__ corner, long long* __restrict__ rec_key,
                   long long* __restrict__ smooth_key) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3ll * F) return;
  const int f = (int)(c / 3), k = (int)(c - 3ll * f), k1 = k == 2 ? 0 : k + 1;
  rec_key[2 * c] = -1;
  rec_key[2 * c + 1] = -1;
  smooth_key[c] = -1;
  if (__ldg(label + f) < 0) return;
  const int a = corner[3ll * f + k], b = corner[3ll * f + k1];
  if (a != b) smooth_key[c] = lv_pair(a, b);
  const int g = __ldg(nbr + c);
  if (g < 0 || f > g || __ldg(label + g) < 0 || __ldg(slot + f) == __ldg(slot + g)) return;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int kk = e ? k1 : k;
    const int vtx = __ldg(faces + 3ll * f + kk);
    int other = -1;
    for (int j = 2; j >= 0; --j)
      if (__ldg(faces + 3ll * g + j) == vtx) other = corner[3ll * g + j];
    rec_key[2 * c + e] = lv_pair(corner[3ll * f + kk], other);
  }
}

struct LvImg {
  const unsigned char* p;
  int W, H;
};

// bilinear at (u, v), pixel centres at integer coordinates, clamped into the image
__device__ __forceinline__ void lv_bilinear(const unsigned char* img, int W, int H, double u,
                                            double v, double out[3]) {
  u = fmin(fmax(u, 0.0), (double)(W - 1));
  v = fmin(fmax(v, 0.0), (double)(H - 1));
  const double fx = floor(u), fy = floor(v);
  const double ax = ds(u, fx), ay = ds(v, fy);
  const int x0 = (int)fx, y0 = (int)fy, x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const double c00 = img[((size_t)y0 * W + x0) * 3 + ch], c10 = img[((size_t)y0 * W + x1) * 3 + ch];
    const double c01 = img[((size_t)y1 * W + x0) * 3 + ch], c11 = img[((size_t)y1 * W + x1) * 3 + ch];
    const double r0 = da(dm(ds(1.0, ax), c00), dm(ax, c10));
    const double r1 = da(dm(ds(1.0, ax), c01), dm(ax, c11));
    out[ch] = da(dm(ds(1.0, ay), r0), dm(ay, r1));
  }
}

__device__ __forceinline__ double lv_row(const float* A, double X, double Y, double Z) {
  return da(da(da(dm((double)A[0], X), dm((double)A[1], Y)), dm((double)A[2], Z)), (double)A[3]);
}

// one thread per endpoint record: SEAM_SAMPLES points from the endpoint toward the other end,
// each sampled in the lower chart's view (a) and the upper chart's view (b), weighted by (1 - t)
__global__ void __launch_bounds__(256)
level_samples_kernel(const float* __restrict__ verts, const int* __restrict__ faces,
                     const int* __restrict__ label, const int* __restrict__ slot,
                     const int* __restrict__ nbr, const long long* __restrict__ rec_sub, int R,
                     const float* __restrict__ Ps, const unsigned long long* __restrict__ images,
                     const int* __restrict__ wh, double* __restrict__ rec) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const long long sub = rec_sub[r];
  const long long c = sub >> 1;
  const int e = (int)(sub & 1);
  const int f = (int)(c / 3), k = (int)(c - 3ll * f), k1 = k == 2 ? 0 : k + 1;
  const int g = __ldg(nbr + c);
  const bool f_low = __ldg(slot + f) < __ldg(slot + g);
  const int va = __ldg(label + (f_low ? f : g)), vb = __ldg(label + (f_low ? g : f));
  const int s0 = __ldg(faces + 3ll * f + (e ? k1 : k)), s1 = __ldg(faces + 3ll * f + (e ? k : k1));
  double x0[3], x1[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    x0[a] = (double)__ldg(verts + 3ll * s0 + a);
    x1[a] = (double)__ldg(verts + 3ll * s1 + a);
  }
  const float* Pa = Ps + (size_t)va * 16;
  const float* Pb = Ps + (size_t)vb * 16;
  const unsigned char* Ia = reinterpret_cast<const unsigned char*>(images[va]);
  const unsigned char* Ib = reinterpret_cast<const unsigned char*>(images[vb]);
  const int Wa = wh[2 * va], Ha = wh[2 * va + 1], Wb = wh[2 * vb], Hb = wh[2 * vb + 1];
  double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int s = 0; s < kLvSamples; ++s) {
    const double t = dd((double)s, (double)kLvSamples);
    const double wt = ds(1.0, t);
    const double X = da(x0[0], dm(t, ds(x1[0], x0[0])));
    const double Y = da(x0[1], dm(t, ds(x1[1], x0[1])));
    const double Z = da(x0[2], dm(t, ds(x1[2], x0[2])));
    double col[3];
    double w = lv_row(Pa + 8, X, Y, Z);
    lv_bilinear(Ia, Wa, Ha, dd(lv_row(Pa, X, Y, Z), w), dd(lv_row(Pa + 4, X, Y, Z), w), col);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) acc[ch] = da(acc[ch], dm(wt, col[ch]));
    w = lv_row(Pb + 8, X, Y, Z);
    lv_bilinear(Ib, Wb, Hb, dd(lv_row(Pb, X, Y, Z), w), dd(lv_row(Pb + 4, X, Y, Z), w), col);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) acc[3 + ch] = da(acc[3 + ch], dm(wt, col[ch]));
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) rec[(size_t)r * 6 + j] = acc[j];
}

// one thread per seam pair: its records in (pair, record) order
__global__ void __launch_bounds__(256)
level_pairs_kernel(const double* __restrict__ rec, const long long* __restrict__ seg, int P,
                   double* __restrict__ fpair) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  double wrec = 0.0;
  for (int s = 0; s < kLvSamples; ++s) wrec = da(wrec, ds(1.0, dd((double)s, (double)kLvSamples)));
  double num[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, den = 0.0;
  for (long long r = seg[p]; r < seg[p + 1]; ++r) {
#pragma unroll
    for (int j = 0; j < 6; ++j) num[j] = da(num[j], rec[(size_t)r * 6 + j]);
    den = da(den, wrec);
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) fpair[(size_t)p * 6 + j] = dd(num[j], den);
}

// ---------------------------------------------------------------- the system
__global__ void __launch_bounds__(256)
level_rowptr_kernel(const long long* __restrict__ ekey, long long nnz, int n,
                    int* __restrict__ rowptr, int* __restrict__ col) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nnz) return;
  const long long k = ekey[i];
  const int row = (int)(k >> 32);
  col[i] = (int)(k & 0xffffffffll);
  if (i == 0 || (int)(ekey[i - 1] >> 32) != row) rowptr[row] = (int)i;
  if (i == nnz - 1) rowptr[n] = (int)nnz;
}

// one thread per row, entries in column order: off-diagonals -1 (seam) or -SMOOTH_WEIGHT
// (smoothing edge), the diagonal -(their sum) + EPS, and the right-hand side
__global__ void __launch_bounds__(256)
level_values_kernel(const int* __restrict__ rowptr, const int* __restrict__ col,
                    const int* __restrict__ etype, int n, const double* __restrict__ fpair,
                    double* __restrict__ val, double* __restrict__ diag, double* __restrict__ rhs) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n) return;
  double s = 0.0, b[3] = {0.0, 0.0, 0.0};
  int di = -1;
  for (int i = rowptr[row]; i < rowptr[row + 1]; ++i) {
    const int t = etype[i];
    if (t == -1) { di = i; continue; }
    const double v = t == -2 ? -kLvSmooth : -1.0;
    val[i] = v;
    s = da(s, v);
    if (t >= 0) {
      const double* fp = fpair + (size_t)t * 6;
      const bool low = row < col[i];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch)
        b[ch] = da(b[ch], low ? ds(fp[3 + ch], fp[ch]) : ds(fp[ch], fp[3 + ch]));
    }
  }
  const double d = da(-s, kLvEps);
  val[di] = d;
  diag[row] = d;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) rhs[(size_t)row * 3 + ch] = b[ch];
}

// ---------------------------------------------------------------- conjugate gradients
struct LvCg {
  double rz[3], bb[3], ratio[3], alpha[3], beta[3];
  int done, iters;
};

// fixed-shape tree over the block of per-thread partials v[Q], into out[blockIdx.x * Q + q]
template <int Q>
__device__ __forceinline__ void lv_block_sum(double (&v)[Q], double* out) {
  __shared__ double sh[Q][kLvThreads];
#pragma unroll
  for (int q = 0; q < Q; ++q) sh[q][threadIdx.x] = v[q];
  __syncthreads();
  for (int w = kLvThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) {
#pragma unroll
      for (int q = 0; q < Q; ++q) sh[q][threadIdx.x] = da(sh[q][threadIdx.x], sh[q][threadIdx.x + w]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int q = 0; q < Q; ++q) out[(size_t)blockIdx.x * Q + q] = sh[q][0];
  }
}

// x = 0, r = b, z = r / d, p = z; partials of r.z and r.r
__global__ void __launch_bounds__(kLvThreads)
level_cg_init_kernel(const double* __restrict__ b, const double* __restrict__ d, int n,
                     double* __restrict__ x, double* __restrict__ r, double* __restrict__ z,
                     double* __restrict__ p, double* __restrict__ part) {
  double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const double di = d[i];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const double ri = b[i * 3 + ch], zi = dd(ri, di);
      x[i * 3 + ch] = 0.0; r[i * 3 + ch] = ri; z[i * 3 + ch] = zi; p[i * 3 + ch] = zi;
      acc[ch] = da(acc[ch], dm(ri, zi));
      acc[3 + ch] = da(acc[3 + ch], dm(ri, ri));
    }
  }
  lv_block_sum<6>(acc, part);
}

// q = A p; partials of p.q
__global__ void __launch_bounds__(kLvThreads)
level_cg_spmv_kernel(const int* __restrict__ rowptr, const int* __restrict__ col,
                     const double* __restrict__ val, int n, const double* __restrict__ p,
                     double* __restrict__ q, double* __restrict__ part, const LvCg* __restrict__ cg) {
  if (cg->done) return;
  double acc[3] = {0.0, 0.0, 0.0};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    double s[3] = {0.0, 0.0, 0.0};
    for (int j = __ldg(rowptr + i); j < __ldg(rowptr + i + 1); ++j) {
      const double a = __ldg(val + j);
      const double* pj = p + (size_t)__ldg(col + j) * 3;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) s[ch] = da(s[ch], dm(a, pj[ch]));
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      q[i * 3 + ch] = s[ch];
      acc[ch] = da(acc[ch], dm(p[i * 3 + ch], s[ch]));
    }
  }
  lv_block_sum<3>(acc, part);
}

// x += alpha p, r -= alpha q, z = r / d; partials of r.z and r.r
__global__ void __launch_bounds__(kLvThreads)
level_cg_update_kernel(const double* __restrict__ d, int n, const double* __restrict__ p,
                       const double* __restrict__ q, double* __restrict__ x, double* __restrict__ r,
                       double* __restrict__ z, double* __restrict__ part, const LvCg* __restrict__ cg) {
  if (cg->done) return;
  const double al[3] = {cg->alpha[0], cg->alpha[1], cg->alpha[2]};
  double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const double di = d[i];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const size_t k = i * 3 + ch;
      x[k] = da(x[k], dm(al[ch], p[k]));
      const double ri = ds(r[k], dm(al[ch], q[k])), zi = dd(ri, di);
      r[k] = ri; z[k] = zi;
      acc[ch] = da(acc[ch], dm(ri, zi));
      acc[3 + ch] = da(acc[3 + ch], dm(ri, ri));
    }
  }
  lv_block_sum<6>(acc, part);
}

// p = z + beta p
__global__ void __launch_bounds__(kLvThreads)
level_cg_direction_kernel(int n, const double* __restrict__ z, double* __restrict__ p,
                          const LvCg* __restrict__ cg) {
  if (cg->done) return;
  const double be[3] = {cg->beta[0], cg->beta[1], cg->beta[2]};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) p[i * 3 + ch] = da(z[i * 3 + ch], dm(be[ch], p[i * 3 + ch]));
}

// one block: the partials of nb blocks summed in a fixed tree; mode 0 = after init (r.z, r.r),
// 1 = after spmv (p.q -> alpha), 2 = after update (r.z, r.r -> ratio, beta, done, iters)
template <int Q>
__global__ void __launch_bounds__(kLvThreads)
level_cg_reduce_kernel(const double* __restrict__ part, int nb, int mode, double tol,
                       LvCg* __restrict__ cg) {
  if (mode != 0 && cg->done) return;
  double acc[Q];
#pragma unroll
  for (int q = 0; q < Q; ++q) acc[q] = 0.0;
  for (int b = threadIdx.x; b < nb; b += blockDim.x)
#pragma unroll
    for (int q = 0; q < Q; ++q) acc[q] = da(acc[q], part[(size_t)b * Q + q]);
  __shared__ double sh[Q][kLvThreads];
#pragma unroll
  for (int q = 0; q < Q; ++q) sh[q][threadIdx.x] = acc[q];
  __syncthreads();
  for (int w = kLvThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) {
#pragma unroll
      for (int q = 0; q < Q; ++q) sh[q][threadIdx.x] = da(sh[q][threadIdx.x], sh[q][threadIdx.x + w]);
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  if constexpr (Q == 3) {
    for (int ch = 0; ch < 3; ++ch) {
      const double pq = sh[ch][0];
      cg->alpha[ch] = pq > 0.0 ? dd(cg->rz[ch], pq) : 0.0;
    }
  } else {
    bool all = true;
    for (int ch = 0; ch < 3; ++ch) {
      const double rz = sh[ch][0], rr = sh[3 + ch][0];
      if (mode == 0) cg->bb[ch] = rr;
      else cg->beta[ch] = cg->rz[ch] > 0.0 ? dd(rz, cg->rz[ch]) : 0.0;
      cg->rz[ch] = rz;
      cg->ratio[ch] = cg->bb[ch] > 0.0 ? dd(__dsqrt_rn(rr), __dsqrt_rn(cg->bb[ch])) : 0.0;
      all = all && cg->ratio[ch] <= tol;
    }
    if (mode == 2) cg->iters += 1;
    if (all) cg->done = 1;
  }
}

// ---------------------------------------------------------------- owners and apply
__device__ __forceinline__ bool lv_face_uv(const float* __restrict__ verts,
                                           const int* __restrict__ faces, int f,
                                           const float* __restrict__ P, double u[3], double v[3]) {
  RenderCam cam;
#pragma unroll
  for (int r = 0; r < 12; ++r) cam.P[r] = P[r];
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int i = __ldg(faces + 3ll * f + k);
    float uf = 0.f, vf = 0.f, wf;
    ok = project(cam, __ldg(verts + 3ll * i), __ldg(verts + 3ll * i + 1), __ldg(verts + 3ll * i + 2),
                 uf, vf, wf) && ok;
    u[k] = uf;
    v[k] = vf;
  }
  return ok;
}

// the point of the triangle (u, v) nearest to (px, py): its distance (0 inside, either winding)
// and barycentrics
__device__ __forceinline__ double lv_nearest(const double u[3], const double v[3], double px,
                                             double py, double l[3]) {
  const double area = ds(dm(ds(u[1], u[0]), ds(v[2], v[0])), dm(ds(v[1], v[0]), ds(u[2], u[0])));
  if (area != 0.0) {
    const double l0 = dd(ds(dm(ds(u[1], px), ds(v[2], py)), dm(ds(v[1], py), ds(u[2], px))), area);
    const double l1 = dd(ds(dm(ds(u[2], px), ds(v[0], py)), dm(ds(v[2], py), ds(u[0], px))), area);
    const double l2 = dd(ds(dm(ds(u[0], px), ds(v[1], py)), dm(ds(v[0], py), ds(u[1], px))), area);
    if (l0 >= 0.0 && l1 >= 0.0 && l2 >= 0.0) {
      l[0] = l0; l[1] = l1; l[2] = l2;
      return 0.0;
    }
  }
  double best = INFINITY, bt = 0.0;
  int bk = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int k1 = k == 2 ? 0 : k + 1;
    const double dx = ds(u[k1], u[k]), dy = ds(v[k1], v[k]);
    const double d2e = da(dm(dx, dx), dm(dy, dy));
    double t = d2e > 0.0 ? dd(da(dm(ds(px, u[k]), dx), dm(ds(py, v[k]), dy)), d2e) : 0.0;
    t = fmin(fmax(t, 0.0), 1.0);
    const double ex = ds(px, da(u[k], dm(t, dx))), ey = ds(py, da(v[k], dm(t, dy)));
    const double d2 = da(dm(ex, ex), dm(ey, ey));
    if (d2 < best) { best = d2; bt = t; bk = k; }
  }
  l[0] = l[1] = l[2] = 0.0;
  l[bk] = ds(1.0, bt);
  l[bk == 2 ? 0 : bk + 1] = bt;
  return __dsqrt_rn(best);
}

// one warp per view-chart face: every integer view pixel of its chart's rectangle within REACH
// of its projected triangle
__global__ void __launch_bounds__(256)
level_owners_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                    const int* __restrict__ label, const int* __restrict__ slot,
                    const int* __restrict__ charts, const float* __restrict__ Ps, int S,
                    unsigned long long* __restrict__ owner) {
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= F) return;
  const int f = (int)wid;
  const int L = __ldg(label + f);
  if (L < 0) return;
  double u[3], v[3];
  if (!lv_face_uv(verts, faces, f, Ps + (size_t)L * 16, u, v)) return;
  const int* c = charts + (size_t)__ldg(slot + f) * 9;
  const int x0 = c[2], y0 = c[3], page = c[6], ox = c[7], oy = c[8];
  const int xlo = max(x0, (int)ceil(ds(fmin(fmin(u[0], u[1]), u[2]), kLvReach)));
  const int xhi = min(c[4], (int)floor(da(fmax(fmax(u[0], u[1]), u[2]), kLvReach)));
  const int ylo = max(y0, (int)ceil(ds(fmin(fmin(v[0], v[1]), v[2]), kLvReach)));
  const int yhi = min(c[5], (int)floor(da(fmax(fmax(v[0], v[1]), v[2]), kLvReach)));
  if (xhi < xlo || yhi < ylo) return;
  const long long nx = xhi - xlo + 1, total = nx * (yhi - ylo + 1);
  unsigned long long* A = owner + (size_t)page * S * S;
  for (long long i = lane; i < total; i += 32) {
    const int y = ylo + (int)(i / nx), x = xlo + (int)(i % nx);
    double l[3];
    const double dist = lv_nearest(u, v, (double)x, (double)y, l);
    if (!(dist <= kLvReach)) continue;
    const unsigned long long key =
        ((unsigned long long)__float_as_uint(__double2float_rn(dist)) << 32) | (unsigned)f;
    atomicMin(A + (size_t)(oy + y - y0) * S + (ox + x - x0), key);
  }
}

__global__ void __launch_bounds__(256)
level_apply_kernel(const unsigned long long* __restrict__ owner, long long n_texels,
                   const float* __restrict__ verts, const int* __restrict__ faces,
                   const int* __restrict__ label, const int* __restrict__ slot,
                   const int* __restrict__ charts, const float* __restrict__ Ps, int S,
                   const int* __restrict__ corner, const double* __restrict__ g,
                   unsigned char* __restrict__ atlas) {
  const long long SS = (long long)S * S;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_texels;
       t += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = owner[t];
    if (key == kKeyEmpty) continue;
    const int f = (int)(key & 0xffffffffull);
    const long long rem = t % SS;
    const int ty = (int)(rem / S), tx = (int)(rem % S);
    const int* c = charts + (size_t)__ldg(slot + f) * 9;
    double u[3], v[3], l[3];
    lv_face_uv(verts, faces, f, Ps + (size_t)__ldg(label + f) * 16, u, v);
    lv_nearest(u, v, (double)(c[2] + tx - c[7]), (double)(c[3] + ty - c[8]), l);
    const int* cu = corner + 3ll * f;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const double off = da(da(dm(l[0], g[(size_t)cu[0] * 3 + ch]), dm(l[1], g[(size_t)cu[1] * 3 + ch])),
                            dm(l[2], g[(size_t)cu[2] * 3 + ch]));
      unsigned char* b = atlas + (size_t)t * 3 + ch;
      *b = (unsigned char)fmin(fmax(rint(da((double)*b, off)), 0.0), 255.0);
    }
  }
}

inline unsigned lv_blocks(long long n) { return (unsigned)((n + 255) / 256); }

inline int lv_cg_blocks(int n) {
  return (int)std::min<long long>(kLvMaxBlocks, std::max<long long>(1, ((long long)n + kLvThreads - 1) / kLvThreads));
}

inline size_t lv_align(size_t b) { return (b + 255) & ~size_t(255); }

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_texture_level_keys(const int* faces, int F, const int* label, const int* slot,
                                         long long* keys, void* stream) {
  const char* what = "texture_level_keys";
  CASMVS_REQUIRE(F >= 0, "%s: F < 0", what);
  if (F == 0) return 0;
  CASMVS_REQUIRE(faces && label && slot && keys, "%s: null pointer", what);
  level_keys_kernel<<<lv_blocks(3ll * F), 256, 0, as_stream(stream)>>>(faces, F, label, slot, keys);
  return after_launch(what);
}

extern "C" int casmvs_texture_level_corners(const long long* keys, int F, const long long* unknowns,
                                            int n, int* corner, void* stream) {
  const char* what = "texture_level_corners";
  CASMVS_REQUIRE(F >= 0 && n >= 0, "%s: F < 0 or n < 0", what);
  if (F == 0) return 0;
  CASMVS_REQUIRE(keys && corner && (n == 0 || unknowns), "%s: null pointer", what);
  level_corners_kernel<<<lv_blocks(3ll * F), 256, 0, as_stream(stream)>>>(keys, F, unknowns, n, corner);
  return after_launch(what);
}

extern "C" int casmvs_texture_level_edges(const int* nbr, const int* faces, int F, const int* label,
                                          const int* slot, const int* corner, long long* rec_key,
                                          long long* smooth_key, void* stream) {
  const char* what = "texture_level_edges";
  CASMVS_REQUIRE(F >= 0, "%s: F < 0", what);
  if (F == 0) return 0;
  CASMVS_REQUIRE(nbr && faces && label && slot && corner && rec_key && smooth_key,
                 "%s: null pointer", what);
  level_edges_kernel<<<lv_blocks(3ll * F), 256, 0, as_stream(stream)>>>(nbr, faces, F, label, slot,
                                                                        corner, rec_key, smooth_key);
  return after_launch(what);
}

extern "C" int casmvs_texture_level_samples(const float* verts, const int* faces, const int* label,
                                            const int* slot, const int* nbr,
                                            const long long* rec_sub, int R, const float* Ps,
                                            const unsigned long long* images, const int* wh,
                                            double* rec, void* stream) {
  const char* what = "texture_level_samples";
  CASMVS_REQUIRE(R >= 0, "%s: R < 0", what);
  if (R == 0) return 0;
  CASMVS_REQUIRE(verts && faces && label && slot && nbr && rec_sub && Ps && images && wh && rec,
                 "%s: null pointer", what);
  level_samples_kernel<<<lv_blocks(R), 256, 0, as_stream(stream)>>>(verts, faces, label, slot, nbr,
                                                                    rec_sub, R, Ps, images, wh, rec);
  return after_launch(what);
}

extern "C" int casmvs_texture_level_pairs(const double* rec, const long long* seg, int P,
                                          double* fpair, void* stream) {
  const char* what = "texture_level_pairs";
  CASMVS_REQUIRE(P >= 0, "%s: P < 0", what);
  if (P == 0) return 0;
  CASMVS_REQUIRE(rec && seg && fpair, "%s: null pointer", what);
  level_pairs_kernel<<<lv_blocks(P), 256, 0, as_stream(stream)>>>(rec, seg, P, fpair);
  return after_launch(what);
}

extern "C" int casmvs_texture_level_system(const long long* ekey, const int* etype, long long nnz,
                                           int n, const double* fpair, int* rowptr, int* col,
                                           double* val, double* diag, double* rhs, void* stream) {
  const char* what = "texture_level_system";
  CASMVS_REQUIRE(n >= 0 && nnz >= n && nnz < (1ll << 31), "%s: need 0 <= n <= nnz < 2^31 (got %d, "
                 "%lld)", what, n, nnz);
  if (n == 0) return 0;
  CASMVS_REQUIRE(ekey && etype && rowptr && col && val && diag && rhs, "%s: null pointer", what);
  cudaStream_t st = as_stream(stream);
  level_rowptr_kernel<<<lv_blocks(nnz), 256, 0, st>>>(ekey, nnz, n, rowptr, col);
  const int rc = after_launch(what);
  if (rc) return rc;
  level_values_kernel<<<lv_blocks(n), 256, 0, st>>>(rowptr, col, etype, n, fpair, val, diag, rhs);
  return after_launch(what);
}

extern "C" size_t casmvs_texture_level_cg_workspace_bytes(int n) {
  if (n <= 0) return 0;
  return 4 * lv_align((size_t)n * 3 * sizeof(double)) +
         lv_align((size_t)lv_cg_blocks(n) * 6 * sizeof(double)) + lv_align(sizeof(LvCg));
}

extern "C" int casmvs_texture_level_cg(const int* rowptr, const int* col, const double* val,
                                       const double* diag, const double* rhs, int n, double* x,
                                       void* workspace, size_t workspace_bytes, int max_iters,
                                       double tol, int check_every, int* iters, double* ratios,
                                       int* converged, void* stream) {
  const char* what = "texture_level_cg";
  CASMVS_REQUIRE(n >= 0 && max_iters >= 0 && check_every >= 1 && tol >= 0.0,
                 "%s: need n >= 0, max_iters >= 0, check_every >= 1, tol >= 0", what);
  CASMVS_REQUIRE(iters && ratios && converged, "%s: null pointer", what);
  *iters = 0;
  *converged = 1;
  ratios[0] = ratios[1] = ratios[2] = 0.0;
  if (n == 0) return 0;
  CASMVS_REQUIRE(rowptr && col && val && diag && rhs && x && workspace, "%s: null pointer", what);
  CASMVS_REQUIRE(workspace_bytes >= casmvs_texture_level_cg_workspace_bytes(n),
                 "%s: workspace of %zu bytes, need %zu", what, workspace_bytes,
                 casmvs_texture_level_cg_workspace_bytes(n));
  const size_t vb = lv_align((size_t)n * 3 * sizeof(double));
  char* w = static_cast<char*>(workspace);
  double *r = (double*)w, *z = (double*)(w + vb), *p = (double*)(w + 2 * vb), *q = (double*)(w + 3 * vb);
  const int nb = lv_cg_blocks(n);
  double* part = (double*)(w + 4 * vb);
  LvCg* cg = (LvCg*)(w + 4 * vb + lv_align((size_t)nb * 6 * sizeof(double)));
  cudaStream_t st = as_stream(stream);
  cudaError_t e = cudaMemsetAsync(cg, 0, sizeof(LvCg), st);
  CASMVS_REQUIRE(e == cudaSuccess, "%s: memset failed: %s", what, cudaGetErrorString(e));
  int rc;
  level_cg_init_kernel<<<nb, kLvThreads, 0, st>>>(rhs, diag, n, x, r, z, p, part);
  if ((rc = after_launch(what))) return rc;
  level_cg_reduce_kernel<6><<<1, kLvThreads, 0, st>>>(part, nb, 0, tol, cg);
  if ((rc = after_launch(what))) return rc;
  LvCg h;
  for (int launched = 0;;) {
    e = cudaMemcpyAsync(&h, cg, sizeof(LvCg), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    CASMVS_REQUIRE(e == cudaSuccess, "%s: %s", what, cudaGetErrorString(e));
    if (h.done || launched >= max_iters) break;
    const int m = std::min(check_every, max_iters - launched);
    for (int it = 0; it < m; ++it, ++launched) {
      level_cg_spmv_kernel<<<nb, kLvThreads, 0, st>>>(rowptr, col, val, n, p, q, part, cg);
      if ((rc = after_launch(what))) return rc;
      level_cg_reduce_kernel<3><<<1, kLvThreads, 0, st>>>(part, nb, 1, tol, cg);
      if ((rc = after_launch(what))) return rc;
      level_cg_update_kernel<<<nb, kLvThreads, 0, st>>>(diag, n, p, q, x, r, z, part, cg);
      if ((rc = after_launch(what))) return rc;
      level_cg_reduce_kernel<6><<<1, kLvThreads, 0, st>>>(part, nb, 2, tol, cg);
      if ((rc = after_launch(what))) return rc;
      level_cg_direction_kernel<<<nb, kLvThreads, 0, st>>>(n, z, p, cg);
      if ((rc = after_launch(what))) return rc;
    }
  }
  *iters = h.iters;
  *converged = h.done;
  for (int ch = 0; ch < 3; ++ch) ratios[ch] = h.ratio[ch];
  return 0;
}

extern "C" int casmvs_texture_level_owners(const float* verts, const int* faces, int F,
                                           const int* label, const int* slot, const int* charts,
                                           const float* Ps, int S, unsigned long long* owner,
                                           void* stream) {
  const char* what = "texture_level_owners";
  CASMVS_REQUIRE(F >= 0 && S >= 4 && S <= kLvMaxSide, "%s: need F >= 0 and S in 4..%d", what,
                 kLvMaxSide);
  if (F == 0) return 0;
  CASMVS_REQUIRE(verts && faces && label && slot && charts && Ps && owner, "%s: null pointer", what);
  level_owners_kernel<<<lv_blocks(32ll * F), 256, 0, as_stream(stream)>>>(verts, faces, F, label,
                                                                          slot, charts, Ps, S, owner);
  return after_launch(what);
}

extern "C" int casmvs_texture_level_apply(const unsigned long long* owner, long long n_texels,
                                          const float* verts, const int* faces, const int* label,
                                          const int* slot, const int* charts, const float* Ps,
                                          int S, const int* corner, const double* g,
                                          unsigned char* atlas, void* stream) {
  const char* what = "texture_level_apply";
  CASMVS_REQUIRE(n_texels >= 0 && S >= 4 && S <= kLvMaxSide, "%s: need n_texels >= 0 and S in "
                 "4..%d", what, kLvMaxSide);
  if (n_texels == 0) return 0;
  CASMVS_REQUIRE(owner && verts && faces && label && slot && charts && Ps && corner && atlas,
                 "%s: null pointer", what);
  const unsigned blocks = (unsigned)std::min<long long>((n_texels + 255) / 256, 132ll * 16);
  level_apply_kernel<<<blocks, 256, 0, as_stream(stream)>>>(owner, n_texels, verts, faces, label,
                                                            slot, charts, Ps, S, corner, g, atlas);
  return after_launch(what);
}
