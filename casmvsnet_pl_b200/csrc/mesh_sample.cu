// Uniform surface sampling of a triangle mesh (casmvsnet_pl_b200/mesh_sample.py drives these;
// oracle/mesh_sample_oracle.py restates them in numpy, bit for bit).  include/casmvs.h states the
// rule.
//
// Every double operation is explicitly rounded (__dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn),
// so nothing is contracted into an FMA, and there are no atomics: each output sample is written
// by exactly one thread, so the same input gives the same bytes on every run.
//
// The points kernel runs one thread per output sample, not per face: a sliver face may hold
// millions of samples.  A thread finds its face by binary search over the exclusive prefix sums
// of the per-face counts (every count is >= 3, so the starts are strictly increasing), within
// the faces of its block's first and last samples, which two threads search for first; then it
// decodes its local index k into the row i and column j of the triangle's lattice with exact
// integer arithmetic: row i starts at R(i) = i (n + 1) - i (i - 1) / 2, and i is the largest
// row with R(i) <= k.  A double estimate from the quadratic's smaller root is corrected by
// integer comparisons, so the result does not depend on the rounding of the estimate.
#include <cmath>

#include "common.cuh"

namespace casmvs {

constexpr double kMaxSampleRows = 65536.0;   // n is clamped here before the integer cast

struct SD3 { double x, y, z; };

__device__ __forceinline__ SD3 sload3(const float* __restrict__ p, long long i) {
  return SD3{(double)__ldg(p + i * 3), (double)__ldg(p + i * 3 + 1), (double)__ldg(p + i * 3 + 2)};
}

__device__ __forceinline__ double edge_len(SD3 p, SD3 q) {
  const double dx = __dsub_rn(q.x, p.x), dy = __dsub_rn(q.y, p.y), dz = __dsub_rn(q.z, p.z);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

__device__ __forceinline__ long long row_start(long long i, long long n) {
  return i * (n + 1) - i * (i - 1) / 2;
}

__global__ void __launch_bounds__(256)
mesh_sample_count_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                         double spacing, int* __restrict__ n_out, long long* __restrict__ count) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const SD3 a = sload3(verts, __ldg(faces + 3 * f)), b = sload3(verts, __ldg(faces + 3 * f + 1)),
            c = sload3(verts, __ldg(faces + 3 * f + 2));
  const double L = fmax(fmax(edge_len(a, b), edge_len(b, c)), edge_len(c, a));
  const double r = fmin(ceil(__ddiv_rn(L, spacing)), kMaxSampleRows);
  const int n = r >= 1.0 ? (int)r : 1;
  n_out[f] = n;
  count[f] = (long long)(n + 1) * (n + 2) / 2;
}

__global__ void __launch_bounds__(256)
mesh_sample_points_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                          const int* __restrict__ n_in, const long long* __restrict__ start,
                          long long S, float* __restrict__ out) {
  // the faces of the block's first and last samples bound every thread's search
  __shared__ int range[2];
  const long long s0 = (long long)blockIdx.x * blockDim.x;
  if (threadIdx.x < 2) {
    const long long t = threadIdx.x == 0 ? s0 : min(s0 + blockDim.x, S) - 1;
    int lo = 0, hi = F - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(start + mid) <= t) lo = mid; else hi = mid - 1;
    }
    range[threadIdx.x] = lo;
  }
  __syncthreads();
  const long long s = s0 + threadIdx.x;
  if (s >= S) return;
  int lo = range[0], hi = range[1];        // the last face with start <= s
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(start + mid) <= s) lo = mid; else hi = mid - 1;
  }
  const int f = lo;
  const long long n = __ldg(n_in + f), k = s - __ldg(start + f);
  const double m = (double)(2 * n + 3);
  long long i = (long long)((m - sqrt(fmax(m * m - 8.0 * (double)k, 0.0))) * 0.5);
  i = i < 0 ? 0 : (i > n ? n : i);
  while (i > 0 && row_start(i, n) > k) --i;
  while (i < n && row_start(i + 1, n) <= k) ++i;
  const long long j = k - row_start(i, n);
  const double u = __ddiv_rn((double)i, (double)n), v = __ddiv_rn((double)j, (double)n);
  const SD3 a = sload3(verts, __ldg(faces + 3 * f)), b = sload3(verts, __ldg(faces + 3 * f + 1)),
            c = sload3(verts, __ldg(faces + 3 * f + 2));
  float* o = out + 3 * s;
  o[0] = __double2float_rn(__dadd_rn(__dadd_rn(a.x, __dmul_rn(u, __dsub_rn(b.x, a.x))),
                                     __dmul_rn(v, __dsub_rn(c.x, a.x))));
  o[1] = __double2float_rn(__dadd_rn(__dadd_rn(a.y, __dmul_rn(u, __dsub_rn(b.y, a.y))),
                                     __dmul_rn(v, __dsub_rn(c.y, a.y))));
  o[2] = __double2float_rn(__dadd_rn(__dadd_rn(a.z, __dmul_rn(u, __dsub_rn(b.z, a.z))),
                                     __dmul_rn(v, __dsub_rn(c.z, a.z))));
}

inline unsigned sample_blocks(long long n, int t = 256) { return (unsigned)((n + t - 1) / t); }

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_mesh_sample_count(const float* verts, const int* faces, int F, double spacing,
                                        int* n, long long* count, void* stream) {
  CASMVS_REQUIRE(F >= 0 && (long long)F * 3 < 0x7fffffffLL, "mesh_sample_count: face count out of range");
  CASMVS_REQUIRE(spacing > 0.0 && std::isfinite(spacing), "mesh_sample_count: spacing must be finite and > 0");
  if (F == 0) return 0;
  CASMVS_REQUIRE(verts && faces && n && count, "mesh_sample_count: null pointer");
  mesh_sample_count_kernel<<<sample_blocks(F), 256, 0, as_stream(stream)>>>(verts, faces, F, spacing,
                                                                            n, count);
  return after_launch("mesh_sample_count");
}

extern "C" int casmvs_mesh_sample_points(const float* verts, const int* faces, int F, const int* n,
                                         const long long* start, long long S, float* out,
                                         void* stream) {
  CASMVS_REQUIRE(F >= 0 && (long long)F * 3 < 0x7fffffffLL, "mesh_sample_points: face count out of range");
  CASMVS_REQUIRE(S >= 0 && S <= 0x7fffffffLL, "mesh_sample_points: sample count out of range");
  if (S == 0) return 0;
  CASMVS_REQUIRE(F > 0, "mesh_sample_points: samples without faces");
  CASMVS_REQUIRE(verts && faces && n && start && out, "mesh_sample_points: null pointer");
  mesh_sample_points_kernel<<<sample_blocks(S), 256, 0, as_stream(stream)>>>(verts, faces, F, n, start,
                                                                             S, out);
  return after_launch("mesh_sample_points");
}
