// Quadric edge-collapse decimation (Garland & Heckbert 1997) in parallel rounds
// (casmvsnet_pl_b200/simplify.py drives these; oracle/simplify_oracle.py restates them in numpy,
// bit for bit).  include/casmvs.h states the rule.
//
// Every double operation is explicitly rounded (__dmul_rn / __dadd_rn / __ddiv_rn, sqrt is
// correctly rounded), so nothing is contracted into an FMA; sums run in a fixed order and the
// only atomics are integer ones (atomicAdd of counts, atomicMin of keys), whose result does not
// depend on order.  The same input gives the same bytes on every run.
//
// Why the selected collapses of one round do not interfere.  key(e) is unique per edge.  m1[v] is
// the least candidate key at v, m2[v] the least m1 over the closed 1-ring of v (v and the
// vertices of its faces); ab is selected when key(ab) = m2[a] = m2[b].  Let ab != cd both be
// selected and suppose c lies in the 1-ring of a.  Then key(ab) = m2[a] <= m1[c] <= key(cd).
// The 1-ring relation is symmetric, so a lies in the 1-ring of c and likewise key(cd) <= key(ab):
// the keys are equal, so ab = cd, a contradiction.  Hence no endpoint of one selected edge lies
// in the 1-ring of an endpoint of another: no face touches two collapses, every face and vertex
// that a collapse reads or writes is its own, and the round equals the collapses applied one
// after the other in any order.  The least candidate key overall equals m2 at both its ends, so
// every round with a candidate collapses at least one edge.
#include "common.cuh"

namespace casmvs {

constexpr int kMaxFan = 32;
constexpr double kBoundaryWeight = 1000.0;
constexpr double kFoldCos = 0.2;
constexpr double kDetEps = 1e-12;
constexpr long long kSimplifyKeyNone = 0x7fffffffffffffffLL;

struct D3 { double x, y, z; };

__device__ __forceinline__ D3 load3(const float* __restrict__ p, long long i) {
  return D3{(double)__ldg(p + i * 3), (double)__ldg(p + i * 3 + 1), (double)__ldg(p + i * 3 + 2)};
}
__device__ __forceinline__ D3 sub3(D3 a, D3 b) {
  return D3{__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y), __dsub_rn(a.z, b.z)};
}
__device__ __forceinline__ D3 cross3(D3 u, D3 v) {
  return D3{__dsub_rn(__dmul_rn(u.y, v.z), __dmul_rn(u.z, v.y)),
            __dsub_rn(__dmul_rn(u.z, v.x), __dmul_rn(u.x, v.z)),
            __dsub_rn(__dmul_rn(u.x, v.y), __dmul_rn(u.y, v.x))};
}
__device__ __forceinline__ double dot3(D3 u, D3 v) {
  return __dadd_rn(__dadd_rn(__dmul_rn(u.x, v.x), __dmul_rn(u.y, v.y)), __dmul_rn(u.z, v.z));
}

// w [n^, -n^.p0][n^, -n^.p0]^T, n^ = n / |n|, as 10 unique entries (row-major upper triangle)
__device__ __forceinline__ void plane_quadric(D3 n, D3 p0, double w, double q[10]) {
  const double ln = sqrt(dot3(n, n));
  const D3 nh{__ddiv_rn(n.x, ln), __ddiv_rn(n.y, ln), __ddiv_rn(n.z, ln)};
  const double pl[4] = {nh.x, nh.y, nh.z, -dot3(nh, p0)};
  int k = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i; j < 4; ++j) q[k++] = __dmul_rn(w, __dmul_rn(pl[i], pl[j]));
}

__device__ __forceinline__ D3 face_normal(const float* __restrict__ verts, const int* __restrict__ faces,
                                          int f) {
  const D3 p0 = load3(verts, __ldg(faces + 3 * f)), p1 = load3(verts, __ldg(faces + 3 * f + 1)),
           p2 = load3(verts, __ldg(faces + 3 * f + 2));
  return cross3(sub3(p1, p0), sub3(p2, p0));
}

__device__ __forceinline__ double qform(const double q[10], double x, double y, double z) {
  const double u0 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], x), __dmul_rn(q[1], y)), __dmul_rn(q[2], z)), q[3]);
  const double u1 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[1], x), __dmul_rn(q[4], y)), __dmul_rn(q[5], z)), q[6]);
  const double u2 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[2], x), __dmul_rn(q[5], y)), __dmul_rn(q[7], z)), q[8]);
  const double u3 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[3], x), __dmul_rn(q[6], y)), __dmul_rn(q[8], z)), q[9]);
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(u0, x), __dmul_rn(u1, y)), __dmul_rn(u2, z)), u3);
}

__device__ __forceinline__ double det3(double m00, double m01, double m02, double m10, double m11,
                                       double m12, double m20, double m21, double m22) {
  const double t0 = __dmul_rn(m00, __dsub_rn(__dmul_rn(m11, m22), __dmul_rn(m12, m21)));
  const double t1 = __dmul_rn(m01, __dsub_rn(__dmul_rn(m10, m22), __dmul_rn(m12, m20)));
  const double t2 = __dmul_rn(m02, __dsub_rn(__dmul_rn(m10, m21), __dmul_rn(m11, m20)));
  return __dadd_rn(__dsub_rn(t0, t1), t2);
}

__device__ __forceinline__ bool has_vertex(const int* __restrict__ faces, int f, int v) {
  return __ldg(faces + 3 * f) == v || __ldg(faces + 3 * f + 1) == v || __ldg(faces + 3 * f + 2) == v;
}

// ---------------------------------------------------------------------------- input cleanup
__global__ void __launch_bounds__(256)
simplify_clean_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                      unsigned char* __restrict__ keep) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int i0 = __ldg(faces + 3 * f), i1 = __ldg(faces + 3 * f + 1), i2 = __ldg(faces + 3 * f + 2);
  bool ok = i0 != i1 && i1 != i2 && i0 != i2;
  if (ok) {
    const D3 n = face_normal(verts, faces, f);
    ok = !(n.x == 0.0 && n.y == 0.0 && n.z == 0.0);
  }
  keep[f] = ok;
}

__global__ void __launch_bounds__(256)
simplify_frozen_kernel(const int* __restrict__ faces, int V, const int* __restrict__ off,
                       const int* __restrict__ corners, const int* __restrict__ corner_edge,
                       const int* __restrict__ edge_count, unsigned char* __restrict__ frozen) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int o = __ldg(off + v), n = __ldg(off + v + 1) - o;
  if (n > kMaxFan) { frozen[v] = 1; return; }
  int p[kMaxFan], q[kMaxFan];
  for (int i = 0; i < n; ++i) {
    const int c = __ldg(corners + o + i), f = c / 3, k = c - 3 * f;
    if (__ldg(edge_count + __ldg(corner_edge + c)) > 2 ||
        __ldg(edge_count + __ldg(corner_edge + 3 * f + (k + 2) % 3)) > 2) {
      frozen[v] = 1;
      return;
    }
    p[i] = __ldg(faces + 3 * f + (k + 1) % 3);
    q[i] = __ldg(faces + 3 * f + (k + 2) % 3);
  }
  // the faces form one fan when the link graph (edge p-q per face) is connected
  unsigned reached = n ? 1u : 0u;
  const unsigned all = n == 32 ? 0xffffffffu : ((1u << n) - 1u);
  bool grew = true;
  while (grew && reached != all) {
    grew = false;
    for (int i = 0; i < n; ++i) {
      if (reached >> i & 1u) continue;
      for (int j = 0; j < n; ++j)
        if ((reached >> j & 1u) && (p[i] == p[j] || p[i] == q[j] || q[i] == p[j] || q[i] == q[j])) {
          reached |= 1u << i;
          grew = true;
          break;
        }
    }
  }
  frozen[v] = reached != all;
}

// ---------------------------------------------------------------------------- quadrics
__global__ void __launch_bounds__(256)
simplify_face_quadrics_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                              double* __restrict__ fq) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const D3 n = face_normal(verts, faces, f);
  double q[10];
  plane_quadric(n, load3(verts, __ldg(faces + 3 * f)), __dmul_rn(sqrt(dot3(n, n)), 0.5), q);
#pragma unroll
  for (int i = 0; i < 10; ++i) fq[(size_t)f * 10 + i] = q[i];
}

__global__ void __launch_bounds__(256)
simplify_vertex_quadrics_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int V,
                                const int* __restrict__ off, const int* __restrict__ corners,
                                const int* __restrict__ corner_edge,
                                const long long* __restrict__ edge_keys,
                                const int* __restrict__ edge_count, const double* __restrict__ fq,
                                double* __restrict__ Q) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int o = __ldg(off + v), n = __ldg(off + v + 1) - o;
  double s[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) s[i] = 0.0;
  for (int j = 0; j < n; ++j) {
    const int f = __ldg(corners + o + j) / 3;
#pragma unroll
    for (int i = 0; i < 10; ++i) s[i] = __dadd_rn(s[i], __ldg(fq + (size_t)f * 10 + i));
  }
  // boundary edges at v, in increasing edge index (= key order)
  int last = -1;
  for (;;) {
    int best = 0x7fffffff, bf = -1;
    for (int j = 0; j < n; ++j) {
      const int c = __ldg(corners + o + j), f = c / 3, k = c - 3 * f;
      const int e0 = __ldg(corner_edge + c), e1 = __ldg(corner_edge + 3 * f + (k + 2) % 3);
      if (e0 > last && e0 < best && __ldg(edge_count + e0) == 1) { best = e0; bf = f; }
      if (e1 > last && e1 < best && __ldg(edge_count + e1) == 1) { best = e1; bf = f; }
    }
    if (bf < 0) break;
    const long long key = __ldg(edge_keys + best);
    const D3 pa = load3(verts, key >> 32), pb = load3(verts, key & 0xffffffffLL);
    const D3 e = sub3(pb, pa);
    double q[10];
    plane_quadric(cross3(e, face_normal(verts, faces, bf)), pa, __dmul_rn(kBoundaryWeight, dot3(e, e)), q);
#pragma unroll
    for (int i = 0; i < 10; ++i) s[i] = __dadd_rn(s[i], q[i]);
    last = best;
  }
#pragma unroll
  for (int i = 0; i < 10; ++i) Q[(size_t)v * 10 + i] = s[i];
}

// ---------------------------------------------------------------------------- one round
__global__ void __launch_bounds__(256)
simplify_vertex_info_kernel(const long long* __restrict__ edge_keys, const int* __restrict__ edge_count,
                            int E, int* __restrict__ deg, unsigned char* __restrict__ bnd) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const long long key = __ldg(edge_keys + e);
  const int a = (int)(key >> 32), b = (int)(key & 0xffffffffLL);
  atomicAdd(deg + a, 1);
  atomicAdd(deg + b, 1);
  if (__ldg(edge_count + e) == 1) { bnd[a] = 1; bnd[b] = 1; }    // every writer stores 1
}

// Optimal position (Cramer) or the first cheapest of a, b, midpoint; cost in double at the
// float32 position, NaN when it is NaN.
__device__ void position_cost(const double q[10], D3 pa, D3 pb, float v[3], float& cost) {
  const double a00 = q[0], a01 = q[1], a02 = q[2], a11 = q[4], a12 = q[5], a22 = q[7];
  const double r0 = -q[3], r1 = -q[6], r2 = -q[8];
  const double det = det3(a00, a01, a02, a01, a11, a12, a02, a12, a22);
  const double m = fmax(fmax(fmax(fabs(a00), fabs(a01)), fmax(fabs(a02), fabs(a11))),
                        fmax(fabs(a12), fabs(a22)));
  const float x0 = __double2float_rn(__ddiv_rn(det3(r0, a01, a02, r1, a11, a12, r2, a12, a22), det));
  const float x1 = __double2float_rn(__ddiv_rn(det3(a00, r0, a02, a01, r1, a12, a02, r2, a22), det));
  const float x2 = __double2float_rn(__ddiv_rn(det3(a00, a01, r0, a01, a11, r1, a02, a12, r2), det));
  const bool solve = fabs(det) > __dmul_rn(kDetEps, __dmul_rn(__dmul_rn(m, m), m)) &&
                     isfinite(x0) && isfinite(x1) && isfinite(x2);
  if (solve) {
    v[0] = x0; v[1] = x1; v[2] = x2;
  } else {
    const float m0 = __double2float_rn(__dmul_rn(__dadd_rn(pa.x, pb.x), 0.5));
    const float m1 = __double2float_rn(__dmul_rn(__dadd_rn(pa.y, pb.y), 0.5));
    const float m2 = __double2float_rn(__dmul_rn(__dadd_rn(pa.z, pb.z), 0.5));
    const double ca = qform(q, pa.x, pa.y, pa.z), cb = qform(q, pb.x, pb.y, pb.z);
    const double cm = qform(q, m0, m1, m2);
    if (ca <= cb && ca <= cm) { v[0] = (float)pa.x; v[1] = (float)pa.y; v[2] = (float)pa.z; }
    else if (cb <= cm)        { v[0] = (float)pb.x; v[1] = (float)pb.y; v[2] = (float)pb.z; }
    else                      { v[0] = m0; v[1] = m1; v[2] = m2; }
  }
  const double c = qform(q, v[0], v[1], v[2]);
  cost = isnan(c) ? __int_as_float(0x7fc00000) : (c > 0.0 ? __double2float_rn(c) : 0.f);
}

// The topological and geometric conditions of include/casmvs.h for edge ab (neither frozen).
__device__ bool collapse_ok(int a, int b, int cnt, D3 vn, const float* __restrict__ verts,
                            const int* __restrict__ faces, const int* __restrict__ off,
                            const int* __restrict__ corners, const int* __restrict__ deg,
                            const unsigned char* __restrict__ bnd) {
  const int oa = __ldg(off + a), na = __ldg(off + a + 1) - oa;
  const int ob = __ldg(off + b), nb = __ldg(off + b + 1) - ob;
  const bool ba = bnd[a], bb = bnd[b];
  if (ba && bb && cnt != 1) return false;
  if (na + nb - cnt > kMaxFan) return false;
  int opp[2], nopp = 0;
  for (int i = 0; i < na; ++i) {
    const int f = __ldg(corners + oa + i) / 3;
    if (!has_vertex(faces, f, b)) continue;
    int c = -1;
    for (int k = 0; k < 3; ++k) {
      const int w = __ldg(faces + 3 * f + k);
      if (w != a && w != b) c = w;
    }
    if (nopp == 0 || (nopp == 1 && opp[0] != c)) opp[nopp++] = c;
    if (deg[c] - 1 < (bnd[c] ? 2 : 3)) return false;
  }
  // common neighbours of a and b: each neighbour w of a at its first face, looked up around b
  int ncommon = 0;
  for (int i = 0; i < na; ++i) {
    const int f = __ldg(corners + oa + i) / 3;
    for (int k = 0; k < 3; ++k) {
      const int w = __ldg(faces + 3 * f + k);
      if (w == a || w == b) continue;
      bool dup = false;
      for (int j = 0; j < i && !dup; ++j) dup = has_vertex(faces, __ldg(corners + oa + j) / 3, w);
      if (dup) continue;
      for (int j = 0; j < nb; ++j)
        if (has_vertex(faces, __ldg(corners + ob + j) / 3, w)) { ++ncommon; break; }
    }
  }
  if (ncommon != nopp) return false;
  if (deg[a] + deg[b] - 2 - ncommon < (ba || bb ? 2 : 3)) return false;
  // no surviving face around a or b folds
  for (int s = 0; s < 2; ++s) {
    const int u = s ? b : a, o = s ? ob : oa, n = s ? nb : na;
    for (int i = 0; i < n; ++i) {
      const int c = __ldg(corners + o + i), f = c / 3, k = c - 3 * f;
      if (has_vertex(faces, f, s ? a : b)) continue;
      D3 p[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) p[j] = load3(verts, __ldg(faces + 3 * f + j));
      const D3 no = cross3(sub3(p[1], p[0]), sub3(p[2], p[0]));
      if (k == 0) p[0] = vn; else if (k == 1) p[1] = vn; else p[2] = vn;
      const D3 nn = cross3(sub3(p[1], p[0]), sub3(p[2], p[0]));
      if (!(dot3(nn, no) > __dmul_rn(__dmul_rn(kFoldCos, sqrt(dot3(nn, nn))), sqrt(dot3(no, no)))))
        return false;
    }
  }
  return true;
}

__global__ void __launch_bounds__(128)
simplify_edge_costs_kernel(const float* __restrict__ verts, const double* __restrict__ Q,
                           const int* __restrict__ faces, const int* __restrict__ off,
                           const int* __restrict__ corners, const long long* __restrict__ edge_keys,
                           const int* __restrict__ edge_count, int E,
                           const unsigned char* __restrict__ frozen, const int* __restrict__ deg,
                           const unsigned char* __restrict__ bnd, int has_max_error, double max_error,
                           float* __restrict__ newpos, float* __restrict__ cost_out,
                           unsigned char* __restrict__ valid0, long long* __restrict__ key_out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const long long key = __ldg(edge_keys + e);
  const int a = (int)(key >> 32), b = (int)(key & 0xffffffffLL);
  double q[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) q[i] = __dadd_rn(__ldg(Q + (size_t)a * 10 + i), __ldg(Q + (size_t)b * 10 + i));
  float v[3], cost;
  position_cost(q, load3(verts, a), load3(verts, b), v, cost);
  newpos[(size_t)e * 3] = v[0]; newpos[(size_t)e * 3 + 1] = v[1]; newpos[(size_t)e * 3 + 2] = v[2];
  cost_out[e] = cost;
  const bool ok = !frozen[a] && !frozen[b] && isfinite(cost) &&
                  collapse_ok(a, b, __ldg(edge_count + e), D3{v[0], v[1], v[2]}, verts, faces, off,
                              corners, deg, bnd);
  valid0[e] = ok;
  const bool valid = ok && (!has_max_error || (double)cost <= max_error);
  key_out[e] = valid ? ((long long)__float_as_uint(cost) << 32) | e : kSimplifyKeyNone;
}

__global__ void __launch_bounds__(256)
simplify_fill_kernel(long long* __restrict__ x, int n, long long value) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = value;
}

__global__ void __launch_bounds__(256)
simplify_m1_kernel(const long long* __restrict__ edge_keys, const long long* __restrict__ key, int E,
                   long long thr, long long* __restrict__ m1) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const long long k = __ldg(key + e);
  if (k > thr) return;
  const long long ek = __ldg(edge_keys + e);
  atomicMin(reinterpret_cast<unsigned long long*>(m1 + (ek >> 32)), (unsigned long long)k);
  atomicMin(reinterpret_cast<unsigned long long*>(m1 + (ek & 0xffffffffLL)), (unsigned long long)k);
}

__global__ void __launch_bounds__(256)
simplify_m2_kernel(const long long* __restrict__ m1, const int* __restrict__ faces, int V,
                   const int* __restrict__ off, const int* __restrict__ corners,
                   long long* __restrict__ m2) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  long long m = __ldg(m1 + v);
  for (int j = __ldg(off + v); j < __ldg(off + v + 1); ++j) {
    const int f = __ldg(corners + j) / 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) m = min(m, __ldg(m1 + __ldg(faces + 3 * f + k)));
  }
  m2[v] = m;
}

__global__ void __launch_bounds__(256)
simplify_select_kernel(const long long* __restrict__ edge_keys, const long long* __restrict__ key, int E,
                       long long thr, const long long* __restrict__ m2, unsigned char* __restrict__ sel) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const long long k = __ldg(key + e), ek = __ldg(edge_keys + e);
  sel[e] = k <= thr && k == __ldg(m2 + (ek >> 32)) && k == __ldg(m2 + (ek & 0xffffffffLL));
}

__global__ void __launch_bounds__(256)
simplify_collapse_kernel(const long long* __restrict__ edge_keys, const long long* __restrict__ idx,
                         int n, const float* __restrict__ newpos, float* __restrict__ verts,
                         unsigned char* __restrict__ colours, double* __restrict__ Q,
                         int* __restrict__ remap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long e = __ldg(idx + i), key = __ldg(edge_keys + e);
  const int a = (int)(key >> 32), b = (int)(key & 0xffffffffLL);
  const float v[3] = {__ldg(newpos + e * 3), __ldg(newpos + e * 3 + 1), __ldg(newpos + e * 3 + 2)};
  const D3 pa = load3(verts, a), pb = load3(verts, b), ed = sub3(pb, pa);
  const double den = dot3(ed, ed);
  double t = den > 0.0 ? __ddiv_rn(dot3(sub3(D3{v[0], v[1], v[2]}, pa), ed), den) : 0.0;
  t = fmin(fmax(t, 0.0), 1.0);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double c0 = colours[(size_t)a * 3 + c], c1 = colours[(size_t)b * 3 + c];
    const double x = rint(__dadd_rn(c0, __dmul_rn(t, __dsub_rn(c1, c0))));
    colours[(size_t)a * 3 + c] = (unsigned char)fmin(255.0, fmax(0.0, x));
  }
#pragma unroll
  for (int j = 0; j < 10; ++j) Q[(size_t)a * 10 + j] = __dadd_rn(Q[(size_t)a * 10 + j], Q[(size_t)b * 10 + j]);
#pragma unroll
  for (int j = 0; j < 3; ++j) verts[(size_t)a * 3 + j] = v[j];
  remap[b] = a;
}

__global__ void __launch_bounds__(256)
simplify_remap_faces_kernel(int* __restrict__ faces, int F, const int* __restrict__ map,
                            unsigned char* __restrict__ keep) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int i0 = __ldg(map + faces[3 * f]), i1 = __ldg(map + faces[3 * f + 1]), i2 = __ldg(map + faces[3 * f + 2]);
  faces[3 * f] = i0; faces[3 * f + 1] = i1; faces[3 * f + 2] = i2;
  keep[f] = i0 != i1 && i1 != i2 && i0 != i2;
}

__global__ void __launch_bounds__(256)
simplify_mark_used_kernel(const int* __restrict__ faces, int F, int* __restrict__ used) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < 3 * F) used[__ldg(faces + c)] = 1;          // every writer stores 1
}

inline unsigned simplify_blocks(size_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }

}  // namespace casmvs

using namespace casmvs;

#define SIMPLIFY_DIMS(what, n) \
  CASMVS_REQUIRE((n) >= 0 && (long long)(n) * 3 < 0x7fffffffLL, what ": count out of range")

extern "C" int casmvs_simplify_clean(const float* verts, const int* faces, int F,
                                     unsigned char* keep, void* stream) {
  SIMPLIFY_DIMS("simplify_clean", F);
  if (F == 0) return 0;
  CASMVS_REQUIRE(verts && faces && keep, "simplify_clean: null pointer");
  simplify_clean_kernel<<<simplify_blocks(F), 256, 0, as_stream(stream)>>>(verts, faces, F, keep);
  return after_launch("simplify_clean");
}

extern "C" int casmvs_simplify_frozen(const int* faces, int V, const int* off, const int* corners,
                                      const int* corner_edge, const int* edge_count,
                                      unsigned char* frozen, void* stream) {
  SIMPLIFY_DIMS("simplify_frozen", V);
  if (V == 0) return 0;
  CASMVS_REQUIRE(faces && off && corners && corner_edge && edge_count && frozen,
                 "simplify_frozen: null pointer");
  simplify_frozen_kernel<<<simplify_blocks(V), 256, 0, as_stream(stream)>>>(
      faces, V, off, corners, corner_edge, edge_count, frozen);
  return after_launch("simplify_frozen");
}

extern "C" int casmvs_simplify_face_quadrics(const float* verts, const int* faces, int F, double* fq,
                                             void* stream) {
  SIMPLIFY_DIMS("simplify_face_quadrics", F);
  if (F == 0) return 0;
  CASMVS_REQUIRE(verts && faces && fq, "simplify_face_quadrics: null pointer");
  simplify_face_quadrics_kernel<<<simplify_blocks(F), 256, 0, as_stream(stream)>>>(verts, faces, F, fq);
  return after_launch("simplify_face_quadrics");
}

extern "C" int casmvs_simplify_vertex_quadrics(const float* verts, const int* faces, int V,
                                               const int* off, const int* corners,
                                               const int* corner_edge, const long long* edge_keys,
                                               const int* edge_count, const double* fq, double* Q,
                                               void* stream) {
  SIMPLIFY_DIMS("simplify_vertex_quadrics", V);
  if (V == 0) return 0;
  CASMVS_REQUIRE(verts && faces && off && corners && corner_edge && edge_keys && edge_count && fq && Q,
                 "simplify_vertex_quadrics: null pointer");
  simplify_vertex_quadrics_kernel<<<simplify_blocks(V), 256, 0, as_stream(stream)>>>(
      verts, faces, V, off, corners, corner_edge, edge_keys, edge_count, fq, Q);
  return after_launch("simplify_vertex_quadrics");
}

extern "C" int casmvs_simplify_edge_costs(const float* verts, const double* Q, const int* faces, int V,
                                          const int* off, const int* corners,
                                          const long long* edge_keys, const int* edge_count, int E,
                                          const unsigned char* frozen, int has_max_error,
                                          double max_error, int* deg, unsigned char* bnd,
                                          float* newpos, float* cost, unsigned char* valid0,
                                          long long* key, void* stream) {
  SIMPLIFY_DIMS("simplify_edge_costs", V);
  SIMPLIFY_DIMS("simplify_edge_costs", E);
  if (E == 0) return 0;
  CASMVS_REQUIRE(verts && Q && faces && off && corners && edge_keys && edge_count && frozen && deg &&
                 bnd && newpos && cost && valid0 && key, "simplify_edge_costs: null pointer");
  cudaStream_t s = as_stream(stream);
  cudaError_t err = cudaMemsetAsync(deg, 0, (size_t)V * sizeof(int), s);
  if (err == cudaSuccess) err = cudaMemsetAsync(bnd, 0, (size_t)V, s);
  CASMVS_REQUIRE(err == cudaSuccess, "simplify_edge_costs: memset failed: %s", cudaGetErrorString(err));
  simplify_vertex_info_kernel<<<simplify_blocks(E), 256, 0, s>>>(edge_keys, edge_count, E, deg, bnd);
  int rc = after_launch("simplify_vertex_info");
  if (rc) return rc;
  simplify_edge_costs_kernel<<<simplify_blocks(E, 128), 128, 0, s>>>(
      verts, Q, faces, off, corners, edge_keys, edge_count, E, frozen, deg, bnd, has_max_error,
      max_error, newpos, cost, valid0, key);
  return after_launch("simplify_edge_costs");
}

extern "C" int casmvs_simplify_select(const long long* edge_keys, const long long* key, int E,
                                      long long thr, const int* faces, int V, const int* off,
                                      const int* corners, long long* m1, long long* m2,
                                      unsigned char* sel, void* stream) {
  SIMPLIFY_DIMS("simplify_select", V);
  SIMPLIFY_DIMS("simplify_select", E);
  if (E == 0 || V == 0) return 0;
  CASMVS_REQUIRE(edge_keys && key && faces && off && corners && m1 && m2 && sel,
                 "simplify_select: null pointer");
  cudaStream_t s = as_stream(stream);
  simplify_fill_kernel<<<simplify_blocks(V), 256, 0, s>>>(m1, V, kSimplifyKeyNone);
  int rc = after_launch("simplify_fill");
  if (rc) return rc;
  simplify_m1_kernel<<<simplify_blocks(E), 256, 0, s>>>(edge_keys, key, E, thr, m1);
  if ((rc = after_launch("simplify_m1"))) return rc;
  simplify_m2_kernel<<<simplify_blocks(V), 256, 0, s>>>(m1, faces, V, off, corners, m2);
  if ((rc = after_launch("simplify_m2"))) return rc;
  simplify_select_kernel<<<simplify_blocks(E), 256, 0, s>>>(edge_keys, key, E, thr, m2, sel);
  return after_launch("simplify_select");
}

extern "C" int casmvs_simplify_collapse(const long long* edge_keys, const long long* idx, int n,
                                        const float* newpos, float* verts, unsigned char* colours,
                                        double* Q, int* remap, void* stream) {
  SIMPLIFY_DIMS("simplify_collapse", n);
  if (n == 0) return 0;
  CASMVS_REQUIRE(edge_keys && idx && newpos && verts && colours && Q && remap,
                 "simplify_collapse: null pointer");
  simplify_collapse_kernel<<<simplify_blocks(n), 256, 0, as_stream(stream)>>>(
      edge_keys, idx, n, newpos, verts, colours, Q, remap);
  return after_launch("simplify_collapse");
}

extern "C" int casmvs_simplify_remap_faces(int* faces, int F, const int* map, unsigned char* keep,
                                           void* stream) {
  SIMPLIFY_DIMS("simplify_remap_faces", F);
  if (F == 0) return 0;
  CASMVS_REQUIRE(faces && map && keep, "simplify_remap_faces: null pointer");
  simplify_remap_faces_kernel<<<simplify_blocks(F), 256, 0, as_stream(stream)>>>(faces, F, map, keep);
  return after_launch("simplify_remap_faces");
}

extern "C" int casmvs_simplify_mark_used(const int* faces, int F, int V, int* used, void* stream) {
  SIMPLIFY_DIMS("simplify_mark_used", F);
  SIMPLIFY_DIMS("simplify_mark_used", V);
  if (V == 0) return 0;
  CASMVS_REQUIRE(used && (faces || F == 0), "simplify_mark_used: null pointer");
  cudaError_t err = cudaMemsetAsync(used, 0, (size_t)V * sizeof(int), as_stream(stream));
  CASMVS_REQUIRE(err == cudaSuccess, "simplify_mark_used: memset failed: %s", cudaGetErrorString(err));
  if (F == 0) return 0;
  simplify_mark_used_kernel<<<simplify_blocks((size_t)F * 3), 256, 0, as_stream(stream)>>>(faces, F, used);
  return after_launch("simplify_mark_used");
}
