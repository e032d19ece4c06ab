// Mesh cleaning: piece areas, boundary loops and minimum-area hole filling
// (casmvsnet_pl_b200/mesh_clean.py drives these; oracle/mesh_clean_oracle.py restates them in
// numpy, bit for bit).  include/casmvs.h states the rule.
//
// Every double operation is explicitly rounded (__dmul_rn / __dadd_rn / __dsub_rn, sqrt is
// correctly rounded), so nothing is contracted into an FMA.  Piece areas are summed in face order
// by one thread per chunk of faces and then one thread per piece over its chunks, the hole DP's minimum over split indices is a lexicographic (cost,
// index) minimum whose result does not depend on the order lanes combine, and the only atomics
// are integer ones.  The same input gives the same bytes on every run.
#include "common.cuh"

namespace casmvs {

constexpr int kCleanMaxHole = 128;
constexpr double kHoleAreaFraction = 0.1;
constexpr int kFillThreads = 256;
constexpr unsigned char kDiagonalTaken = 255;   // split-table mark: the diagonal is a mesh edge

struct CD3 { double x, y, z; };

__device__ __forceinline__ CD3 cload3(const float* __restrict__ p, long long i) {
  return CD3{(double)__ldg(p + i * 3), (double)__ldg(p + i * 3 + 1), (double)__ldg(p + i * 3 + 2)};
}
__device__ __forceinline__ CD3 csub3(CD3 a, CD3 b) {
  return CD3{__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y), __dsub_rn(a.z, b.z)};
}
__device__ __forceinline__ CD3 ccross3(CD3 u, CD3 v) {
  return CD3{__dsub_rn(__dmul_rn(u.y, v.z), __dmul_rn(u.z, v.y)),
             __dsub_rn(__dmul_rn(u.z, v.x), __dmul_rn(u.x, v.z)),
             __dsub_rn(__dmul_rn(u.x, v.y), __dmul_rn(u.y, v.x))};
}
__device__ __forceinline__ double cdot3(CD3 u, CD3 v) {
  return __dadd_rn(__dadd_rn(__dmul_rn(u.x, v.x), __dmul_rn(u.y, v.y)), __dmul_rn(u.z, v.z));
}
__device__ __forceinline__ double clean_inf() { return __longlong_as_double(0x7ff0000000000000LL); }

// ---------------------------------------------------------------------------- pieces
__global__ void __launch_bounds__(256)
mesh_clean_face_area_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                            double* __restrict__ area) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const CD3 p0 = cload3(verts, __ldg(faces + 3 * f)), p1 = cload3(verts, __ldg(faces + 3 * f + 1)),
            p2 = cload3(verts, __ldg(faces + 3 * f + 2));
  const CD3 n = ccross3(csub3(p1, p0), csub3(p2, p0));
  area[f] = __dmul_rn(0.5, sqrt(cdot3(n, n)));
}

__global__ void __launch_bounds__(256)
mesh_clean_sums_kernel(const double* __restrict__ value, const long long* __restrict__ order,
                       const long long* __restrict__ start, int n, double* __restrict__ out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  double s = 0.0;
  for (long long i = __ldg(start + p); i < __ldg(start + p + 1); ++i)
    s = __dadd_rn(s, __ldg(value + (order ? __ldg(order + i) : i)));
  out[p] = s;
}

// ---------------------------------------------------------------------------- boundary loops
__global__ void __launch_bounds__(256)
mesh_clean_degree_kernel(const int* __restrict__ faces, int F, const int* __restrict__ corner_edge,
                         const int* __restrict__ edge_count, int* __restrict__ out_deg,
                         int* __restrict__ in_deg) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3LL * F) return;
  if (__ldg(edge_count + __ldg(corner_edge + c)) != 1) return;
  const long long f = c / 3, k = c - 3 * f;
  atomicAdd(out_deg + __ldg(faces + c), 1);
  atomicAdd(in_deg + __ldg(faces + 3 * f + (k + 1) % 3), 1);
}

// next[a] = b only where a has one boundary half-edge out and one in: its only writer.
__global__ void __launch_bounds__(256)
mesh_clean_next_kernel(const int* __restrict__ faces, int F, const int* __restrict__ corner_edge,
                       const int* __restrict__ edge_count, const int* __restrict__ out_deg,
                       const int* __restrict__ in_deg, int* __restrict__ next,
                       int* __restrict__ next_face) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3LL * F) return;
  if (__ldg(edge_count + __ldg(corner_edge + c)) != 1) return;
  const long long f = c / 3, k = c - 3 * f;
  const int a = __ldg(faces + c);
  if (__ldg(out_deg + a) != 1 || __ldg(in_deg + a) != 1) return;
  next[a] = __ldg(faces + 3 * f + (k + 1) % 3);
  next_face[a] = (int)f;
}

__global__ void __launch_bounds__(256)
mesh_clean_loop_sizes_kernel(const int* __restrict__ next, const int* __restrict__ comp, int V,
                             int* __restrict__ size, unsigned char* __restrict__ open) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int w = __ldg(next + v);
  if (w < 0) return;
  const int r = __ldg(comp + v);
  atomicAdd(size + r, 1);
  if (__ldg(next + w) < 0) open[r] = 1;                 // every writer stores 1
}

// ---------------------------------------------------------------------------- hole filling
__device__ __forceinline__ bool has_edge(const long long* __restrict__ keys, int E, int a, int b) {
  const long long key = ((long long)min(a, b) << 32) | (long long)max(a, b);
  int lo = 0, hi = E;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo < E && __ldg(keys + lo) == key;
}

// One CTA per loop of n = size[L] <= 128 positions.  Shared memory: cost (n, n) double, the loop's
// points (n, 3) double, its vertices (n) int32 and the split table (n, n) u8.
__global__ void __launch_bounds__(kFillThreads)
mesh_clean_fill_kernel(const float* __restrict__ verts, const int* __restrict__ next,
                       const int* __restrict__ next_face, const int* __restrict__ owner,
                       const int* __restrict__ size, const long long* __restrict__ tri_off,
                       const long long* __restrict__ edge_keys, int E,
                       const double* __restrict__ piece_area, unsigned char* __restrict__ status,
                       double* __restrict__ area_out, int* __restrict__ tris) {
  extern __shared__ __align__(16) unsigned char clean_smem[];
  const int L = blockIdx.x, n = __ldg(size + L), o = __ldg(owner + L);
  double* cost = reinterpret_cast<double*>(clean_smem);
  double* P = cost + n * n;
  int* vid = reinterpret_cast<int*>(P + 3 * n);
  unsigned char* split = reinterpret_cast<unsigned char*>(vid + n);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = kFillThreads / 32;
  if (tid == 0) {
    int v = o;
    for (int i = 0; i < n; ++i) { vid[i] = v; v = __ldg(next + v); }
  }
  __syncthreads();
  for (int i = tid; i < n; i += kFillThreads) {
    const CD3 p = cload3(verts, vid[i]);
    P[3 * i] = p.x; P[3 * i + 1] = p.y; P[3 * i + 2] = p.z;
  }
  // cost[i][i+1] = 0; a diagonal (j >= i + 2, not the closing edge 0 -- n-1) that is already a
  // mesh edge marks its cell
  for (int idx = tid; idx < n * n; idx += kFillThreads) {
    const int i = idx / n, j = idx - i * n;
    if (j == i + 1) cost[idx] = 0.0;
    else if (j >= i + 2)
      split[idx] = (!(i == 0 && j == n - 1) && has_edge(edge_keys, E, vid[i], vid[j])) ? kDiagonalTaken : 0;
  }
  __syncthreads();
  const double inf = clean_inf();
  for (int d = 2; d < n; ++d) {
    for (int i = warp; i + d < n; i += nwarps) {
      const int j = i + d;
      double best = inf;
      int bk = n;
      if (split[i * n + j] != kDiagonalTaken) {
        const CD3 pi{P[3 * i], P[3 * i + 1], P[3 * i + 2]}, pj{P[3 * j], P[3 * j + 1], P[3 * j + 2]};
        const CD3 ej = csub3(pj, pi);
        for (int k = i + 1 + lane; k < j; k += 32) {
          const CD3 pk{P[3 * k], P[3 * k + 1], P[3 * k + 2]};
          const CD3 nn = ccross3(csub3(pk, pi), ej);
          if (nn.x == 0.0 && nn.y == 0.0 && nn.z == 0.0) continue;
          const double c = __dadd_rn(__dadd_rn(cost[i * n + k], cost[k * n + j]),
                                     __dmul_rn(0.5, sqrt(cdot3(nn, nn))));
          if (c < best) { best = c; bk = k; }
        }
      }
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, s);
        const int ok = __shfl_xor_sync(0xffffffffu, bk, s);
        if (ob < best || (ob == best && ok < bk)) { best = ob; bk = ok; }
      }
      if (lane == 0) {
        cost[i * n + j] = best;
        split[i * n + j] = (unsigned char)(bk < n ? bk : kDiagonalTaken);
      }
    }
    __syncthreads();
  }
  if (tid != 0) return;
  const double total = cost[n - 1];
  int* out = tris + tri_off[L] * 3;
  area_out[L] = total;
  if (!(total < inf)) {
    status[L] = 2;
    for (int t = 0; t < 3 * (n - 2); ++t) out[t] = -1;
    return;
  }
  status[L] = total <= __dmul_rn(kHoleAreaFraction, __ldg(piece_area + __ldg(next_face + o))) ? 1 : 3;
  // pre-order, left part first: (i, j) emits (j, k, i), then (i, k), then (k, j)
  unsigned char st[2 * kCleanMaxHole];
  int top = 0, t = 0;
  st[top++] = 0; st[top++] = (unsigned char)(n - 1);
  while (top) {
    const int j = st[--top], i = st[--top];
    if (j - i < 2) continue;
    const int k = split[i * n + j];
    out[3 * t] = vid[j]; out[3 * t + 1] = vid[k]; out[3 * t + 2] = vid[i];
    ++t;
    st[top++] = (unsigned char)k; st[top++] = (unsigned char)j;
    st[top++] = (unsigned char)i; st[top++] = (unsigned char)k;
  }
}

inline unsigned clean_blocks(long long n, int t = 256) { return (unsigned)((n + t - 1) / t); }

inline size_t fill_smem_bytes(int n) { return (size_t)n * n * 9 + (size_t)n * 28; }

}  // namespace casmvs

using namespace casmvs;

#define CLEAN_DIMS(what, n) \
  CASMVS_REQUIRE((n) >= 0 && (long long)(n) * 3 < 0x7fffffffLL, what ": count out of range")

extern "C" int casmvs_mesh_clean_face_area(const float* verts, const int* faces, int F, double* area,
                                           void* stream) {
  CLEAN_DIMS("mesh_clean_face_area", F);
  if (F == 0) return 0;
  CASMVS_REQUIRE(verts && faces && area, "mesh_clean_face_area: null pointer");
  mesh_clean_face_area_kernel<<<clean_blocks(F), 256, 0, as_stream(stream)>>>(verts, faces, F, area);
  return after_launch("mesh_clean_face_area");
}

extern "C" int casmvs_mesh_clean_sums(const double* value, const long long* order,
                                      const long long* start, int n, double* out, void* stream) {
  CLEAN_DIMS("mesh_clean_sums", n);
  if (n == 0) return 0;
  CASMVS_REQUIRE(value && start && out, "mesh_clean_sums: null pointer");
  mesh_clean_sums_kernel<<<clean_blocks(n), 256, 0, as_stream(stream)>>>(value, order, start, n, out);
  return after_launch("mesh_clean_sums");
}

extern "C" int casmvs_mesh_clean_boundary(const int* faces, int F, const int* corner_edge,
                                          const int* edge_count, int V, int* out_deg, int* in_deg,
                                          int* next, int* next_face, void* stream) {
  CLEAN_DIMS("mesh_clean_boundary", F);
  CLEAN_DIMS("mesh_clean_boundary", V);
  if (V == 0) return 0;
  CASMVS_REQUIRE(out_deg && in_deg && next && next_face && (F == 0 || (faces && corner_edge && edge_count)),
                 "mesh_clean_boundary: null pointer");
  cudaStream_t s = as_stream(stream);
  cudaError_t err = cudaMemsetAsync(out_deg, 0, (size_t)V * sizeof(int), s);
  if (err == cudaSuccess) err = cudaMemsetAsync(in_deg, 0, (size_t)V * sizeof(int), s);
  if (err == cudaSuccess) err = cudaMemsetAsync(next, 0xff, (size_t)V * sizeof(int), s);
  if (err == cudaSuccess) err = cudaMemsetAsync(next_face, 0xff, (size_t)V * sizeof(int), s);
  CASMVS_REQUIRE(err == cudaSuccess, "mesh_clean_boundary: memset failed: %s", cudaGetErrorString(err));
  if (F == 0) return 0;
  mesh_clean_degree_kernel<<<clean_blocks(3LL * F), 256, 0, s>>>(faces, F, corner_edge, edge_count,
                                                                 out_deg, in_deg);
  int rc = after_launch("mesh_clean_degree");
  if (rc) return rc;
  mesh_clean_next_kernel<<<clean_blocks(3LL * F), 256, 0, s>>>(faces, F, corner_edge, edge_count,
                                                               out_deg, in_deg, next, next_face);
  return after_launch("mesh_clean_next");
}

extern "C" int casmvs_mesh_clean_loop_sizes(const int* next, const int* comp, int V, int* size,
                                            unsigned char* open, void* stream) {
  CLEAN_DIMS("mesh_clean_loop_sizes", V);
  if (V == 0) return 0;
  CASMVS_REQUIRE(next && comp && size && open, "mesh_clean_loop_sizes: null pointer");
  cudaStream_t s = as_stream(stream);
  cudaError_t err = cudaMemsetAsync(size, 0, (size_t)V * sizeof(int), s);
  if (err == cudaSuccess) err = cudaMemsetAsync(open, 0, (size_t)V, s);
  CASMVS_REQUIRE(err == cudaSuccess, "mesh_clean_loop_sizes: memset failed: %s", cudaGetErrorString(err));
  mesh_clean_loop_sizes_kernel<<<clean_blocks(V), 256, 0, s>>>(next, comp, V, size, open);
  return after_launch("mesh_clean_loop_sizes");
}

extern "C" int casmvs_mesh_clean_fill(const float* verts, const int* next, const int* next_face,
                                      const int* owner, const int* size, int n_loops, int max_size,
                                      const long long* tri_off, const long long* edge_keys, int E,
                                      const double* piece_area, unsigned char* status,
                                      double* area, int* tris, void* stream) {
  const char* what = "mesh_clean_fill";
  CASMVS_REQUIRE(n_loops >= 0 && E >= 0, "%s: counts out of range", what);
  if (n_loops == 0) return 0;
  CASMVS_REQUIRE(max_size >= 3 && max_size <= kCleanMaxHole,
                 "%s: loop sizes must lie in 3..%d (got a largest of %d)", what, kCleanMaxHole, max_size);
  CASMVS_REQUIRE(verts && next && next_face && owner && size && tri_off && edge_keys && piece_area &&
                 status && area && tris, "%s: null pointer", what);
  static std::atomic<bool> opted[kMaxDevices];
  int rc = opt_in_smem(mesh_clean_fill_kernel, (int)fill_smem_bytes(kCleanMaxHole), opted, what);
  if (rc) return rc;
  mesh_clean_fill_kernel<<<n_loops, kFillThreads, fill_smem_bytes(max_size), as_stream(stream)>>>(
      verts, next, next_face, owner, size, tri_off, edge_keys, E, piece_area, status, area, tris);
  return after_launch(what);
}
