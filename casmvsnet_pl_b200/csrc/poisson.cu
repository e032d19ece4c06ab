// Poisson surface reconstruction of an oriented (or camera-oriented) point cloud on a dense node
// grid (casmvsnet_pl_b200/poisson.py drives these; oracle/poisson_oracle.py restates them in
// numpy float64).  The surface is extracted by mesh.cu's marching cubes.
//
// Grid: N = 2^depth nodes per axis, node spacing h; local node (x, y, z) = global node lo + (x,
// y, z), at world (lo + x) h.  Dense fields are flat, index (x N + y) N + z.  A point's cell is
// the node round(p / h) (float division); its splat corners are floor(p / h) + {0,1}^3.
//
// No float atomics anywhere: every sum walks its terms in a fixed order (points in sorted cell
// order, neighbour cells x-major, reductions by a fixed tree), so a run's bits do not depend on
// scheduling.
#include "common.cuh"

namespace casmvs {

constexpr long long kPoissonKeyNone = 0x7fffffffffffffffLL;
constexpr int kBias = 1 << 20;                // mesh.cu's brick key offset per axis
constexpr int kSumThreads = 256;
constexpr double kRankEps = 1e-10;            // rank < 2: lambda_mid <= kRankEps * lambda_max

inline unsigned pblocks(size_t n) { return (unsigned)((n + 255) / 256); }

__device__ __forceinline__ size_t node(int x, int y, int z, int N) {
  return ((size_t)x * N + y) * N + z;
}
__device__ __forceinline__ void node_xyz(size_t i, int N, int& x, int& y, int& z) {
  z = (int)(i % N);
  y = (int)((i / N) % N);
  x = (int)(i / ((size_t)N * N));
}

// Fixed-tree block sum of one double per thread (blockDim.x == kSumThreads).
__device__ double block_sum(double v) {
  __shared__ double sh[kSumThreads];
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kSumThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  return sh[0];
}

// One block: thread t sums partials t, t + 1024, ... in order, then a fixed tree.
__global__ void __launch_bounds__(1024) poisson_sum_partials_kernel(const double* __restrict__ part,
                                                                  int n, double* __restrict__ out) {
  __shared__ double sh[1024];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += 1024) s += part[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int k = 512; k > 0; k >>= 1) {
    if ((int)threadIdx.x < k) sh[threadIdx.x] += sh[threadIdx.x + k];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = sh[0];
}

// ---------------------------------------------------------------------------- cells and normals
__global__ void __launch_bounds__(256)
poisson_cell_keys_kernel(const float* __restrict__ pts, const float* __restrict__ nin, int n, float h,
                         int lx, int ly, int lz, int N, long long* __restrict__ keys,
                         float* __restrict__ nout) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int lo[3] = {lx, ly, lz};
  int c[3];
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float q = rintf(__fdiv_rn(__ldg(pts + (size_t)i * 3 + a), h));
    ok = ok && fabsf(q) < 1e9f;                 // false for NaN and inf
    c[a] = ok ? (int)q - lo[a] : 0;
    ok = ok && c[a] >= 0 && c[a] < N;
  }
  if (nin) {
    const double x = __ldg(nin + (size_t)i * 3), y = __ldg(nin + (size_t)i * 3 + 1),
                 z = __ldg(nin + (size_t)i * 3 + 2);
    const double L = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
    const bool nok = L > 0.0 && L < INFINITY;
    ok = ok && nok;
    nout[(size_t)i * 3] = nok ? (float)(x / L) : 0.f;
    nout[(size_t)i * 3 + 1] = nok ? (float)(y / L) : 0.f;
    nout[(size_t)i * 3 + 2] = nok ? (float)(z / L) : 0.f;
  }
  keys[i] = ok ? ((long long)c[0] * N + c[1]) * N + c[2] : kPoissonKeyNone;
}

// moments[c] = count, sum d (3), sum d d^T (xx, xy, xz, yy, yz, zz), d = p - centre, in double,
// over the cell's points in sorted order
__global__ void __launch_bounds__(256)
poisson_cell_moments_kernel(const float* __restrict__ pts, const int* __restrict__ start, int nc,
                            double cx, double cy, double cz, double* __restrict__ mom) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  double m[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = __ldg(start + c); j < __ldg(start + c + 1); ++j) {
    const double x = (double)__ldg(pts + (size_t)j * 3) - cx;
    const double y = (double)__ldg(pts + (size_t)j * 3 + 1) - cy;
    const double z = (double)__ldg(pts + (size_t)j * 3 + 2) - cz;
    m[0] += 1.0;
    m[1] += x; m[2] += y; m[3] += z;
    m[4] += x * x; m[5] += x * y; m[6] += x * z; m[7] += y * y; m[8] += y * z; m[9] += z * z;
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) mom[(size_t)c * 10 + k] = m[k];
}

// One Jacobi rotation zeroing a[p][q] of a symmetric 3x3 matrix (v accumulates the rotations).
template <int p, int q>
__device__ __forceinline__ bool jacobi_rotate(double (&a)[3][3], double (&v)[3][3]) {
  const double apq = a[p][q];
  if (fabs(apq) <= 1e-300 || fabs(apq) <= 1e-18 * (fabs(a[p][p]) + fabs(a[q][q]))) return false;
  const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
  const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double akp = a[k][p], akq = a[k][q];
    a[k][p] = c * akp - s * akq;
    a[k][q] = s * akp + c * akq;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double apk = a[p][k], aqk = a[q][k];
    a[p][k] = c * apk - s * aqk;
    a[q][k] = s * apk + c * aqk;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double vkp = v[k][p], vkq = v[k][q];
    v[k][p] = c * vkp - s * vkq;
    v[k][q] = s * vkp + c * vkq;
  }
  return true;
}

// Cyclic Jacobi on a symmetric 3x3 matrix: a -> diagonal, v's columns the eigenvectors.
__device__ void jacobi3(double (&a)[3][3], double (&v)[3][3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int k = 0; k < 3; ++k) v[r][k] = r == k ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 32; ++sweep) {
    bool rotated = jacobi_rotate<0, 1>(a, v);
    rotated |= jacobi_rotate<0, 2>(a, v);
    rotated |= jacobi_rotate<1, 2>(a, v);
    if (!rotated) break;
  }
}

__global__ void __launch_bounds__(128)
poisson_cell_normals_kernel(const long long* __restrict__ ckeys, const int* __restrict__ cell_of,
                            const double* __restrict__ mom, int nc, int N,
                            double* __restrict__ cn, unsigned char* __restrict__ cok) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  const long long k = __ldg(ckeys + c);
  const int x = (int)(k / ((long long)N * N)), y = (int)((k / N) % N), z = (int)(k % N);
  double m[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int dx = -1; dx <= 1; ++dx)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dz = -1; dz <= 1; ++dz) {
        const int X = x + dx, Y = y + dy, Z = z + dz;
        if (X < 0 || Y < 0 || Z < 0 || X >= N || Y >= N || Z >= N) continue;
        const int o = __ldg(cell_of + node(X, Y, Z, N));
        if (o < 0) continue;
#pragma unroll
        for (int j = 0; j < 10; ++j) m[j] += __ldg(mom + (size_t)o * 10 + j);
      }
  double nrm[3] = {0, 0, 0};
  bool ok = m[0] >= 3.0;
  if (ok) {
    const double mx = m[1] / m[0], my = m[2] / m[0], mz = m[3] / m[0];
    double a[3][3], v[3][3];
    a[0][0] = m[4] / m[0] - mx * mx; a[0][1] = m[5] / m[0] - mx * my; a[0][2] = m[6] / m[0] - mx * mz;
    a[1][1] = m[7] / m[0] - my * my; a[1][2] = m[8] / m[0] - my * mz; a[2][2] = m[9] / m[0] - mz * mz;
    a[1][0] = a[0][1]; a[2][0] = a[0][2]; a[2][1] = a[1][2];
    jacobi3(a, v);
    // eigenvalues in ascending order (l0 <= l1 <= l2); column k0 belongs to l0
    const double d0 = a[0][0], d1 = a[1][1], d2 = a[2][2];
    const int k0 = d0 <= d1 ? (d0 <= d2 ? 0 : 2) : (d1 <= d2 ? 1 : 2);
    const double l0 = fmin(d0, fmin(d1, d2)), l2 = fmax(d0, fmax(d1, d2));
    const double l1 = fmax(fmin(d0, d1), fmin(fmax(d0, d1), d2));
    ok = l2 > 0.0 && l1 > kRankEps * l2;
    const double e0 = k0 == 0 ? v[0][0] : k0 == 1 ? v[0][1] : v[0][2];
    const double e1 = k0 == 0 ? v[1][0] : k0 == 1 ? v[1][1] : v[1][2];
    const double e2 = k0 == 0 ? v[2][0] : k0 == 1 ? v[2][1] : v[2][2];
    const double L = sqrt(e0 * e0 + e1 * e1 + e2 * e2);
    nrm[0] = e0 / L; nrm[1] = e1 / L; nrm[2] = e2 / L;
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) cn[(size_t)c * 3 + j] = ok ? nrm[j] : 0.0;
  cok[c] = ok;
}

// n . (C - p) > 0 for the nearest camera centre C (the first of equal distances)
__global__ void __launch_bounds__(256)
poisson_orient_kernel(const float* __restrict__ pts, const int* __restrict__ pcell,
                      const double* __restrict__ cn, int n, const double* __restrict__ cams, int ncam,
                      float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double px = __ldg(pts + (size_t)i * 3), py = __ldg(pts + (size_t)i * 3 + 1),
               pz = __ldg(pts + (size_t)i * 3 + 2);
  double best = INFINITY;
  int kb = 0;
  for (int k = 0; k < ncam; ++k) {
    const double dx = px - __ldg(cams + k * 3), dy = py - __ldg(cams + k * 3 + 1),
                 dz = pz - __ldg(cams + k * 3 + 2);
    const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    if (d2 < best) { best = d2; kb = k; }
  }
  const int c = __ldg(pcell + i);
  double nx = __ldg(cn + (size_t)c * 3), ny = __ldg(cn + (size_t)c * 3 + 1),
         nz = __ldg(cn + (size_t)c * 3 + 2);
  const double dot = nx * (__ldg(cams + kb * 3) - px) + ny * (__ldg(cams + kb * 3 + 1) - py) +
                     nz * (__ldg(cams + kb * 3 + 2) - pz);
  if (dot < 0.0) { nx = -nx; ny = -ny; nz = -nz; }
  out[(size_t)i * 3] = (float)nx;
  out[(size_t)i * 3 + 1] = (float)ny;
  out[(size_t)i * 3 + 2] = (float)nz;
}

// ---------------------------------------------------------------------------- splat
// float32 trilinear weight of the corner d of a point: (wx wy) wz, w = frac or 1 - frac
__device__ __forceinline__ float corner_weight(float fx, float fy, float fz, int dx, int dy, int dz) {
  const float wx = dx ? fx : __fsub_rn(1.f, fx);
  const float wy = dy ? fy : __fsub_rn(1.f, fy);
  const float wz = dz ? fz : __fsub_rn(1.f, fz);
  return __fmul_rn(__fmul_rn(wx, wy), wz);
}
__device__ __forceinline__ int point_axis(const float* __restrict__ pts, size_t j, int a, float h,
                                          int lo, float& fr) {
  const float q = __fdiv_rn(__ldg(pts + j * 3 + a), h);
  const float fl = floorf(q);
  fr = __fsub_rn(q, fl);
  return (int)fl - lo;
}

// One thread per node gathers the points of the 27 cells around it (a point in cell c has its
// floor corner in c - {0,1}^3), so each node sums its own contributions in sorted order.
__global__ void __launch_bounds__(256)
poisson_splat_kernel(const float* __restrict__ pts, const float* __restrict__ nrm,
                     const unsigned char* __restrict__ rgb, const int* __restrict__ start,
                     const int* __restrict__ cell_of, int N, float h, int lx, int ly, int lz,
                     float* __restrict__ V, float* __restrict__ W, float* __restrict__ C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)N * N * N) return;
  int x, y, z;
  node_xyz(i, N, x, y, z);
  double v0 = 0, v1 = 0, v2 = 0, w = 0, c0 = 0, c1 = 0, c2 = 0;
#pragma unroll 1
  for (int t = 0; t < 27; ++t) {                // cells x-major, then y, then z
    const int cx = x + t / 9 - 1, cy = y + (t / 3) % 3 - 1, cz = z + t % 3 - 1;
    if (cx < 0 || cy < 0 || cz < 0 || cx >= N || cy >= N || cz >= N) continue;
    const int c = __ldg(cell_of + node(cx, cy, cz, N));
    if (c < 0) continue;
    const int j1 = __ldg(start + c + 1);
    for (int j = __ldg(start + c); j < j1; ++j) {
      float fx, fy, fz;
      const int dx = x - point_axis(pts, j, 0, h, lx, fx);
      const int dy = y - point_axis(pts, j, 1, h, ly, fy);
      const int dz = z - point_axis(pts, j, 2, h, lz, fz);
      if ((unsigned)dx > 1u || (unsigned)dy > 1u || (unsigned)dz > 1u) continue;
      const double wt = corner_weight(fx, fy, fz, dx, dy, dz);
      w += wt;
      v0 += wt * __ldg(nrm + (size_t)j * 3);
      v1 += wt * __ldg(nrm + (size_t)j * 3 + 1);
      v2 += wt * __ldg(nrm + (size_t)j * 3 + 2);
      if (rgb) {
        c0 += wt * rgb[(size_t)j * 3];
        c1 += wt * rgb[(size_t)j * 3 + 1];
        c2 += wt * rgb[(size_t)j * 3 + 2];
      } else {
        c0 += wt * 255.0; c1 += wt * 255.0; c2 += wt * 255.0;
      }
    }
  }
  V[i * 3] = (float)v0; V[i * 3 + 1] = (float)v1; V[i * 3 + 2] = (float)v2;
  W[i] = (float)w;
  C[i * 3] = (float)c0; C[i * 3 + 1] = (float)c1; C[i * 3 + 2] = (float)c2;
}

// ---------------------------------------------------------------------------- right-hand side
__device__ __forceinline__ bool interior(int x, int y, int z, int n) {
  return x > 0 && y > 0 && z > 0 && x < n - 1 && y < n - 1 && z < n - 1;
}

__global__ void __launch_bounds__(kSumThreads)
poisson_rhs_kernel(const float* __restrict__ V, int N, float h, float* __restrict__ b,
                   double* __restrict__ part) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < (size_t)N * N * N) {
    int x, y, z;
    node_xyz(i, N, x, y, z);
    float bf = 0.f;
    if (interior(x, y, z, N)) {
      const size_t sx = (size_t)N * N, sy = N;
      const double d = ((double)__ldg(V + (i + sx) * 3) - __ldg(V + (i - sx) * 3)) +
                       ((double)__ldg(V + (i + sy) * 3 + 1) - __ldg(V + (i - sy) * 3 + 1)) +
                       ((double)__ldg(V + (i + 1) * 3 + 2) - __ldg(V + (i - 1) * 3 + 2));
      bf = (float)(d / (2.0 * (double)h));
    }
    b[i] = bf;
    v = (double)bf * bf;
  }
  const double s = block_sum(v);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// ---------------------------------------------------------------------------- multigrid
// Level l has n = N >> l nodes per axis, node I at fine node 2^l I.  The finest level (l = 0)
// holds chi = 0 on its outer layer (indices 0 and N - 1).  Every coarse level (l > 0) puts its
// upper Dirichlet node at index n, which is fine index N, the same place on every coarse level:
// it is not stored and reads as 0, so the coarse interior is 1..n-1.
template <typename T>
__device__ __forceinline__ T nbsum(const T* __restrict__ e, size_t i, int n) {
  const size_t sx = (size_t)n * n, sy = n;
  return ((((e[i - sx] + e[i + sx]) + e[i - sy]) + e[i + sy]) + e[i - 1]) + e[i + 1];
}
__device__ __forceinline__ bool level_interior(int x, int y, int z, int n, int level) {
  const int top = level ? n : n - 1;
  return x > 0 && y > 0 && z > 0 && x < top && y < top && z < top;
}
// neighbour sum of an interior node of any level; the unstored node at index n reads as 0
template <typename T>
__device__ __forceinline__ T level_nbsum(const T* __restrict__ e, size_t i, int x, int y, int z,
                                         int n) {
  const size_t sx = (size_t)n * n, sy = n;
  const T zx = x + 1 < n ? e[i + sx] : T(0), zy = y + 1 < n ? e[i + sy] : T(0),
          zz = z + 1 < n ? e[i + 1] : T(0);
  return ((((e[i - sx] + zx) + e[i - sy]) + zy) + e[i - 1]) + zz;
}

// r = b - (nbsum(chi) - 6 chi) / h^2 at interior nodes in double, 0 on the outer layer
__global__ void __launch_bounds__(kSumThreads)
poisson_residual_kernel(const double* __restrict__ chi, const float* __restrict__ b, int N, float h,
                        float* __restrict__ r, double* __restrict__ part) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < (size_t)N * N * N) {
    int x, y, z;
    node_xyz(i, N, x, y, z);
    double ri = 0.0;
    if (interior(x, y, z, N)) {
      const double hh = (double)h * h;
      ri = (double)__ldg(b + i) - (nbsum(chi, i, N) - 6.0 * chi[i]) / hh;
    }
    r[i] = (float)ri;
    v = ri * ri;
  }
  const double s = block_sum(v);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// red-black Gauss-Seidel half sweep on (nbsum(e) - 6 e) / h^2 = r: nodes with x+y+z = parity mod 2
__global__ void __launch_bounds__(256)
poisson_smooth_kernel(float* __restrict__ e, const float* __restrict__ r, int n, int level, float h2,
                      int parity) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * n * n) return;
  int x, y, z;
  node_xyz(i, n, x, y, z);
  if (!level_interior(x, y, z, n, level) || ((x + y + z) & 1) != parity) return;
  e[i] = (level_nbsum(e, i, x, y, z, n) - h2 * __ldg(r + i)) / 6.f;
}

// The coarsest grid (n^3 <= 1024 nodes) in one block: e = 0, then `sweeps` red-black sweeps.
__global__ void __launch_bounds__(1024)
poisson_smooth_coarse_kernel(float* __restrict__ e, const float* __restrict__ r, int n, int level,
                             float h2, int sweeps) {
  __shared__ float se[1024];
  const int i = threadIdx.x, nn = n * n * n;
  int x = 0, y = 0, z = 0;
  if (i < nn) node_xyz(i, n, x, y, z);
  const bool in = i < nn && level_interior(x, y, z, n, level);
  const float ri = in ? r[i] : 0.f;
  if (i < nn) se[i] = 0.f;
  __syncthreads();
  for (int s = 0; s < sweeps; ++s)
    for (int parity = 0; parity < 2; ++parity) {
      if (in && ((x + y + z) & 1) == parity) se[i] = (level_nbsum(se, i, x, y, z, n) - h2 * ri) / 6.f;
      __syncthreads();
    }
  if (i < nn) e[i] = se[i];
}

__global__ void __launch_bounds__(256)
poisson_mg_residual_kernel(const float* __restrict__ e, const float* __restrict__ r, int n, int level,
                           float h2, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * n * n) return;
  int x, y, z;
  node_xyz(i, n, x, y, z);
  out[i] = level_interior(x, y, z, n, level)
               ? __ldg(r + i) - (level_nbsum(e, i, x, y, z, n) - 6.f * __ldg(e + i)) / h2
               : 0.f;
}

// full weighting: coarse interior node I (1..nc-1) from fine 2I + {-1,0,1}^3 (all stored: 2I + 1 <=
// nf - 1), weights (1/4, 1/2, 1/4)^3
__global__ void __launch_bounds__(256)
poisson_restrict_kernel(const float* __restrict__ f, int nf, float* __restrict__ c) {
  const int nc = nf / 2;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)nc * nc * nc) return;
  int x, y, z;
  node_xyz(i, nc, x, y, z);
  float s = 0.f;
  if (level_interior(x, y, z, nc, 1)) {
    for (int dx = -1; dx <= 1; ++dx)
      for (int dy = -1; dy <= 1; ++dy)
        for (int dz = -1; dz <= 1; ++dz) {
          const float w = (dx ? 0.25f : 0.5f) * (dy ? 0.25f : 0.5f) * (dz ? 0.25f : 0.5f);
          s += w * __ldg(f + node(2 * x + dx, 2 * y + dy, 2 * z + dz, nf));
        }
  }
  c[i] = s;
}

// fine interior node i (of level fine_level) += trilinear interpolation of the coarse nodes
// (coarse I sits at fine 2I; the unstored coarse node nc counts as 0)
__global__ void __launch_bounds__(256)
poisson_prolong_add_kernel(const float* __restrict__ c, int nc, float* __restrict__ f, int fine_level) {
  const int nf = nc * 2;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)nf * nf * nf) return;
  int p[3];
  node_xyz(i, nf, p[0], p[1], p[2]);
  if (!level_interior(p[0], p[1], p[2], nf, fine_level)) return;
  int i0[3], i1[3];
  float w1[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    i0[a] = p[a] >> 1;
    i1[a] = (p[a] + 1) >> 1;
    w1[a] = (p[a] & 1) ? 0.5f : 0.f;
  }
  float s = 0.f;
  for (int d = 0; d < 8; ++d) {
    const int dx = d >> 2, dy = (d >> 1) & 1, dz = d & 1;
    const float w = (dx ? w1[0] : 1.f - w1[0]) * (dy ? w1[1] : 1.f - w1[1]) * (dz ? w1[2] : 1.f - w1[2]);
    const int X = dx ? i1[0] : i0[0], Y = dy ? i1[1] : i0[1], Z = dz ? i1[2] : i0[2];
    if (w == 0.f || X >= nc || Y >= nc || Z >= nc) continue;
    s += w * __ldg(c + node(X, Y, Z, nc));
  }
  f[i] += s;
}

__global__ void __launch_bounds__(256)
poisson_accumulate_kernel(double* __restrict__ chi, const float* __restrict__ e, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) chi[i] += (double)__ldg(e + i);
}

// ---------------------------------------------------------------------------- iso level
__global__ void __launch_bounds__(kSumThreads)
poisson_iso_kernel(const double* __restrict__ chi, const float* __restrict__ pts, int n, int N,
                   float h, int lx, int ly, int lz, double* __restrict__ part) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (j < n) {
    int b[3];
    float fr[3];
    b[0] = point_axis(pts, j, 0, h, lx, fr[0]);
    b[1] = point_axis(pts, j, 1, h, ly, fr[1]);
    b[2] = point_axis(pts, j, 2, h, lz, fr[2]);
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      const int dx = d >> 2, dy = (d >> 1) & 1, dz = d & 1;
      const int X = b[0] + dx, Y = b[1] + dy, Z = b[2] + dz;
      if ((unsigned)X >= (unsigned)N || (unsigned)Y >= (unsigned)N || (unsigned)Z >= (unsigned)N)
        continue;                             // outside the grid, where chi = 0
      v += (double)corner_weight(fr[0], fr[1], fr[2], dx, dy, dz) * __ldg(chi + node(X, Y, Z, N));
    }
  }
  const double s = block_sum(v);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// ---------------------------------------------------------------------------- trim and bricks
// out = 1 where any of the nodes within `radius` along `axis` is set in `in` (or W > 0 when in
// is the float field)
__global__ void __launch_bounds__(256)
poisson_dilate_kernel(const unsigned char* __restrict__ in, const float* __restrict__ Win, int N,
                      int axis, unsigned char* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)N * N * N) return;
  int p[3];
  node_xyz(i, N, p[0], p[1], p[2]);
  const size_t stride = axis == 0 ? (size_t)N * N : axis == 1 ? (size_t)N : 1;
  unsigned char any = 0;
  for (int d = -2; d <= 2; ++d) {
    const int q = p[axis] + d;
    if (q < 0 || q >= N) continue;
    const size_t k = i + (ptrdiff_t)d * (ptrdiff_t)stride;
    any |= Win ? (unsigned char)(__ldg(Win + k) > 0.f) : __ldg(in + k);
  }
  out[i] = any;
}

__device__ __forceinline__ void unpack_brick(long long k, int& bx, int& by, int& bz) {
  bx = (int)(k >> 42) - kBias;
  by = (int)((k >> 21) & 0x1fffff) - kBias;
  bz = (int)(k & 0x1fffff) - kBias;
}

// flags[(i nby + j) nbz + k] = 1 when global brick (b0x + i, b0y + j, b0z + k) holds a kept node
__global__ void __launch_bounds__(256)
poisson_brick_flags_kernel(const unsigned char* __restrict__ keep, int N, int lx, int ly, int lz,
                           int b0x, int b0y, int b0z, int nbx, int nby, int nbz,
                           unsigned char* __restrict__ flags) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)nbx * nby * nbz) return;
  const int k = (int)(t % nbz), j = (int)((t / nbz) % nby), i = (int)(t / ((size_t)nby * nbz));
  const int x0 = (b0x + i) * 8 - lx, y0 = (b0y + j) * 8 - ly, z0 = (b0z + k) * 8 - lz;
  unsigned char any = 0;
  for (int x = max(x0, 0); x < min(x0 + 8, N) && !any; ++x)
    for (int y = max(y0, 0); y < min(y0 + 8, N) && !any; ++y)
      for (int z = max(z0, 0); z < min(z0 + 8, N); ++z)
        if (__ldg(keep + node(x, y, z, N))) { any = 1; break; }
  flags[t] = any;
}

// local node of brick voxel v, false when outside the grid
__device__ __forceinline__ bool voxel_node(const long long* __restrict__ keys, size_t v, int N,
                                           int lx, int ly, int lz, int& x, int& y, int& z) {
  int bx, by, bz;
  unpack_brick(__ldg(keys + (v >> 9)), bx, by, bz);
  const int l = (int)(v & 511);
  x = bx * 8 + (l & 7) - lx;
  y = by * 8 + ((l >> 3) & 7) - ly;
  z = bz * 8 + (l >> 6) - lz;
  return x >= 0 && y >= 0 && z >= 0 && x < N && y < N && z < N;
}

// weight 1 and colour = box5(C) / box5(W) (double sums) at kept nodes; 0 elsewhere
__global__ void __launch_bounds__(256)
poisson_fill_bricks_kernel(const long long* __restrict__ keys, int nb, const unsigned char* __restrict__ keep,
                           const float* __restrict__ W, const float* __restrict__ C, int N, int lx,
                           int ly, int lz, float* __restrict__ weight, float* __restrict__ color) {
  const size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= (size_t)nb * 512) return;
  int x, y, z;
  float wo = 0.f, c[3] = {0.f, 0.f, 0.f};
  if (voxel_node(keys, v, N, lx, ly, lz, x, y, z) && __ldg(keep + node(x, y, z, N))) {
    double sw = 0, s0 = 0, s1 = 0, s2 = 0;
    for (int X = max(x - 2, 0); X <= min(x + 2, N - 1); ++X)
      for (int Y = max(y - 2, 0); Y <= min(y + 2, N - 1); ++Y)
        for (int Z = max(z - 2, 0); Z <= min(z + 2, N - 1); ++Z) {
          const size_t k = node(X, Y, Z, N);
          sw += __ldg(W + k);
          s0 += __ldg(C + k * 3); s1 += __ldg(C + k * 3 + 1); s2 += __ldg(C + k * 3 + 2);
        }
    wo = 1.f;
    c[0] = (float)(s0 / sw); c[1] = (float)(s1 / sw); c[2] = (float)(s2 / sw);
  }
  weight[v] = wo;
  color[v * 3] = c[0]; color[v * 3 + 1] = c[1]; color[v * 3 + 2] = c[2];
}

__global__ void __launch_bounds__(256)
poisson_fill_tsdf_kernel(const long long* __restrict__ keys, int nb, const float* __restrict__ weight,
                         const double* __restrict__ chi, double iso, int N, int lx, int ly, int lz,
                         float* __restrict__ tsdf) {
  const size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= (size_t)nb * 512) return;
  int x, y, z;
  float f = 0.f;
  if (__ldg(weight + v) > 0.f && voxel_node(keys, v, N, lx, ly, lz, x, y, z))
    f = (float)(__ldg(chi + node(x, y, z, N)) - iso);
  tsdf[v] = f;
}

inline int finish_sum(double* part, int nparts, double* out, cudaStream_t st, const char* what) {
  poisson_sum_partials_kernel<<<1, 1024, 0, st>>>(part, nparts, out);
  return after_launch(what);
}

inline bool grid_ok(int N) { return N >= 8 && N <= 1024 && (N & (N - 1)) == 0; }

}  // namespace casmvs

using namespace casmvs;

#define POISSON_GRID(what, N) \
  CASMVS_REQUIRE(grid_ok(N), what ": N must be a power of two in 8..1024, got %d", N)

extern "C" size_t casmvs_poisson_workspace_bytes(long long n) {
  return n <= 0 ? 0 : (size_t)((n + kSumThreads - 1) / kSumThreads) * sizeof(double);
}

extern "C" int casmvs_poisson_cell_keys(const float* points, const float* normals, int n, float h,
                                        int lo_x, int lo_y, int lo_z, int N, long long* keys,
                                        float* unit_normals, void* stream) {
  CASMVS_REQUIRE(n >= 0, "poisson_cell_keys: n < 0");
  CASMVS_REQUIRE(h > 0.f, "poisson_cell_keys: h must be > 0");
  POISSON_GRID("poisson_cell_keys", N);
  if (n == 0) return 0;
  CASMVS_REQUIRE(points && keys && (!normals || unit_normals), "poisson_cell_keys: null pointer");
  poisson_cell_keys_kernel<<<pblocks(n), 256, 0, as_stream(stream)>>>(
      points, normals, n, h, lo_x, lo_y, lo_z, N, keys, unit_normals);
  return after_launch("poisson_cell_keys");
}

extern "C" int casmvs_poisson_cell_moments(const float* points, const int* cell_start, int n_cells,
                                           double cx, double cy, double cz, double* moments,
                                           void* stream) {
  CASMVS_REQUIRE(n_cells >= 0, "poisson_cell_moments: n_cells < 0");
  if (n_cells == 0) return 0;
  CASMVS_REQUIRE(points && cell_start && moments, "poisson_cell_moments: null pointer");
  poisson_cell_moments_kernel<<<pblocks(n_cells), 256, 0, as_stream(stream)>>>(
      points, cell_start, n_cells, cx, cy, cz, moments);
  return after_launch("poisson_cell_moments");
}

extern "C" int casmvs_poisson_cell_normals(const long long* cell_keys, const int* cell_of,
                                           const double* moments, int n_cells, int N,
                                           double* cell_normals, unsigned char* cell_ok, void* stream) {
  CASMVS_REQUIRE(n_cells >= 0, "poisson_cell_normals: n_cells < 0");
  POISSON_GRID("poisson_cell_normals", N);
  if (n_cells == 0) return 0;
  CASMVS_REQUIRE(cell_keys && cell_of && moments && cell_normals && cell_ok,
                 "poisson_cell_normals: null pointer");
  poisson_cell_normals_kernel<<<(n_cells + 127) / 128, 128, 0, as_stream(stream)>>>(
      cell_keys, cell_of, moments, n_cells, N, cell_normals, cell_ok);
  return after_launch("poisson_cell_normals");
}

extern "C" int casmvs_poisson_orient(const float* points, const int* point_cell,
                                     const double* cell_normals, int n, const double* cams,
                                     int n_cams, float* normals, void* stream) {
  CASMVS_REQUIRE(n >= 0 && n_cams >= 1, "poisson_orient: need n >= 0 and at least one camera");
  if (n == 0) return 0;
  CASMVS_REQUIRE(points && point_cell && cell_normals && cams && normals, "poisson_orient: null pointer");
  poisson_orient_kernel<<<pblocks(n), 256, 0, as_stream(stream)>>>(points, point_cell, cell_normals,
                                                                    n, cams, n_cams, normals);
  return after_launch("poisson_orient");
}

extern "C" int casmvs_poisson_splat(const float* points, const float* normals,
                                    const unsigned char* rgb, const int* cell_start,
                                    const int* cell_of, int N, float h, int lo_x, int lo_y, int lo_z,
                                    float* V, float* W, float* C, void* stream) {
  POISSON_GRID("poisson_splat", N);
  CASMVS_REQUIRE(h > 0.f, "poisson_splat: h must be > 0");
  CASMVS_REQUIRE(points && normals && cell_start && cell_of && V && W && C,
                 "poisson_splat: null pointer");
  poisson_splat_kernel<<<pblocks((size_t)N * N * N), 256, 0, as_stream(stream)>>>(
      points, normals, rgb, cell_start, cell_of, N, h, lo_x, lo_y, lo_z, V, W, C);
  return after_launch("poisson_splat");
}

extern "C" int casmvs_poisson_rhs(const float* V, int N, float h, float* b, double* workspace,
                                  double* bb, void* stream) {
  POISSON_GRID("poisson_rhs", N);
  CASMVS_REQUIRE(h > 0.f, "poisson_rhs: h must be > 0");
  CASMVS_REQUIRE(V && b && workspace && bb, "poisson_rhs: null pointer");
  const unsigned nblk = pblocks((size_t)N * N * N);
  poisson_rhs_kernel<<<nblk, kSumThreads, 0, as_stream(stream)>>>(V, N, h, b, workspace);
  const int rc = after_launch("poisson_rhs");
  return rc ? rc : finish_sum(workspace, (int)nblk, bb, as_stream(stream), "poisson_rhs");
}

extern "C" int casmvs_poisson_residual(const double* chi, const float* b, int N, float h, float* r,
                                       double* workspace, double* rr, void* stream) {
  POISSON_GRID("poisson_residual", N);
  CASMVS_REQUIRE(h > 0.f, "poisson_residual: h must be > 0");
  CASMVS_REQUIRE(chi && b && r && workspace && rr, "poisson_residual: null pointer");
  const unsigned nblk = pblocks((size_t)N * N * N);
  poisson_residual_kernel<<<nblk, kSumThreads, 0, as_stream(stream)>>>(chi, b, N, h, r, workspace);
  const int rc = after_launch("poisson_residual");
  return rc ? rc : finish_sum(workspace, (int)nblk, rr, as_stream(stream), "poisson_residual");
}

extern "C" int casmvs_poisson_smooth(float* e, const float* r, int n, int level, float h, int sweeps,
                                     int zero_first, void* stream) {
  POISSON_GRID("poisson_smooth", n);
  CASMVS_REQUIRE(level >= 0, "poisson_smooth: level < 0");
  CASMVS_REQUIRE(h > 0.f && sweeps >= 0, "poisson_smooth: need h > 0 and sweeps >= 0");
  CASMVS_REQUIRE(e && r, "poisson_smooth: null pointer");
  const float h2 = h * h;
  const size_t nn = (size_t)n * n * n;
  if (zero_first && nn <= 1024) {
    poisson_smooth_coarse_kernel<<<1, 1024, 0, as_stream(stream)>>>(e, r, n, level, h2, sweeps);
    return after_launch("poisson_smooth");
  }
  if (zero_first) {
    cudaError_t err = cudaMemsetAsync(e, 0, nn * sizeof(float), as_stream(stream));
    CASMVS_REQUIRE(err == cudaSuccess, "poisson_smooth: memset failed: %s", cudaGetErrorString(err));
  }
  for (int s = 0; s < sweeps; ++s)
    for (int parity = 0; parity < 2; ++parity) {
      poisson_smooth_kernel<<<pblocks(nn), 256, 0, as_stream(stream)>>>(e, r, n, level, h2, parity);
      const int rc = after_launch("poisson_smooth");
      if (rc) return rc;
    }
  return 0;
}

extern "C" int casmvs_poisson_mg_residual(const float* e, const float* r, int n, int level, float h,
                                          float* out, void* stream) {
  POISSON_GRID("poisson_mg_residual", n);
  CASMVS_REQUIRE(level >= 0, "poisson_mg_residual: level < 0");
  CASMVS_REQUIRE(h > 0.f, "poisson_mg_residual: h must be > 0");
  CASMVS_REQUIRE(e && r && out, "poisson_mg_residual: null pointer");
  poisson_mg_residual_kernel<<<pblocks((size_t)n * n * n), 256, 0, as_stream(stream)>>>(
      e, r, n, level, h * h, out);
  return after_launch("poisson_mg_residual");
}

extern "C" int casmvs_poisson_restrict(const float* fine, int nf, float* coarse, void* stream) {
  POISSON_GRID("poisson_restrict", nf);
  CASMVS_REQUIRE(nf >= 16, "poisson_restrict: the fine grid needs >= 16 nodes per axis");
  CASMVS_REQUIRE(fine && coarse, "poisson_restrict: null pointer");
  const size_t nc = nf / 2;
  poisson_restrict_kernel<<<pblocks(nc * nc * nc), 256, 0, as_stream(stream)>>>(fine, nf, coarse);
  return after_launch("poisson_restrict");
}

extern "C" int casmvs_poisson_prolong_add(const float* coarse, int nc, float* fine, int fine_level,
                                          void* stream) {
  POISSON_GRID("poisson_prolong_add", nc);
  CASMVS_REQUIRE(fine_level >= 0, "poisson_prolong_add: fine_level < 0");
  CASMVS_REQUIRE(nc <= 512, "poisson_prolong_add: the coarse grid has at most 512 nodes per axis");
  CASMVS_REQUIRE(coarse && fine, "poisson_prolong_add: null pointer");
  const size_t nf = 2 * (size_t)nc;
  poisson_prolong_add_kernel<<<pblocks(nf * nf * nf), 256, 0, as_stream(stream)>>>(
      coarse, nc, fine, fine_level);
  return after_launch("poisson_prolong_add");
}

extern "C" int casmvs_poisson_accumulate(double* chi, const float* e, int N, void* stream) {
  POISSON_GRID("poisson_accumulate", N);
  CASMVS_REQUIRE(chi && e, "poisson_accumulate: null pointer");
  const size_t nn = (size_t)N * N * N;
  poisson_accumulate_kernel<<<pblocks(nn), 256, 0, as_stream(stream)>>>(chi, e, nn);
  return after_launch("poisson_accumulate");
}

extern "C" int casmvs_poisson_iso_sum(const double* chi, const float* points, int n, int N, float h,
                                      int lo_x, int lo_y, int lo_z, double* workspace, double* sum,
                                      void* stream) {
  POISSON_GRID("poisson_iso_sum", N);
  CASMVS_REQUIRE(n >= 1 && h > 0.f, "poisson_iso_sum: need n >= 1 and h > 0");
  CASMVS_REQUIRE(chi && points && workspace && sum, "poisson_iso_sum: null pointer");
  const unsigned nblk = pblocks(n);
  poisson_iso_kernel<<<nblk, kSumThreads, 0, as_stream(stream)>>>(chi, points, n, N, h, lo_x, lo_y,
                                                                  lo_z, workspace);
  const int rc = after_launch("poisson_iso_sum");
  return rc ? rc : finish_sum(workspace, (int)nblk, sum, as_stream(stream), "poisson_iso_sum");
}

extern "C" int casmvs_poisson_trim(const float* W, int N, unsigned char* keep,
                                   unsigned char* workspace, void* stream) {
  POISSON_GRID("poisson_trim", N);
  CASMVS_REQUIRE(W && keep && workspace, "poisson_trim: null pointer");
  const unsigned nblk = pblocks((size_t)N * N * N);
  cudaStream_t st = as_stream(stream);
  poisson_dilate_kernel<<<nblk, 256, 0, st>>>(nullptr, W, N, 0, keep);
  int rc = after_launch("poisson_trim");
  if (rc) return rc;
  poisson_dilate_kernel<<<nblk, 256, 0, st>>>(keep, nullptr, N, 1, workspace);
  rc = after_launch("poisson_trim");
  if (rc) return rc;
  poisson_dilate_kernel<<<nblk, 256, 0, st>>>(workspace, nullptr, N, 2, keep);
  return after_launch("poisson_trim");
}

extern "C" int casmvs_poisson_brick_flags(const unsigned char* keep, int N, int lo_x, int lo_y,
                                          int lo_z, int b0_x, int b0_y, int b0_z, int nb_x,
                                          int nb_y, int nb_z, unsigned char* flags, void* stream) {
  POISSON_GRID("poisson_brick_flags", N);
  CASMVS_REQUIRE(nb_x > 0 && nb_y > 0 && nb_z > 0, "poisson_brick_flags: empty brick range");
  CASMVS_REQUIRE(keep && flags, "poisson_brick_flags: null pointer");
  poisson_brick_flags_kernel<<<pblocks((size_t)nb_x * nb_y * nb_z), 256, 0, as_stream(stream)>>>(
      keep, N, lo_x, lo_y, lo_z, b0_x, b0_y, b0_z, nb_x, nb_y, nb_z, flags);
  return after_launch("poisson_brick_flags");
}

extern "C" int casmvs_poisson_fill_bricks(const long long* keys, int nb, const unsigned char* keep,
                                          const float* W, const float* C, int N, int lo_x, int lo_y,
                                          int lo_z, float* weight, float* color, void* stream) {
  POISSON_GRID("poisson_fill_bricks", N);
  CASMVS_REQUIRE(nb >= 0, "poisson_fill_bricks: nb < 0");
  if (nb == 0) return 0;
  CASMVS_REQUIRE(keys && keep && W && C && weight && color, "poisson_fill_bricks: null pointer");
  poisson_fill_bricks_kernel<<<pblocks((size_t)nb * 512), 256, 0, as_stream(stream)>>>(
      keys, nb, keep, W, C, N, lo_x, lo_y, lo_z, weight, color);
  return after_launch("poisson_fill_bricks");
}

extern "C" int casmvs_poisson_fill_tsdf(const long long* keys, int nb, const float* weight,
                                        const double* chi, double iso, int N, int lo_x, int lo_y,
                                        int lo_z, float* tsdf, void* stream) {
  POISSON_GRID("poisson_fill_tsdf", N);
  CASMVS_REQUIRE(nb >= 0, "poisson_fill_tsdf: nb < 0");
  if (nb == 0) return 0;
  CASMVS_REQUIRE(keys && weight && chi && tsdf, "poisson_fill_tsdf: null pointer");
  poisson_fill_tsdf_kernel<<<pblocks((size_t)nb * 512), 256, 0, as_stream(stream)>>>(
      keys, nb, weight, chi, iso, N, lo_x, lo_y, lo_z, tsdf);
  return after_launch("poisson_fill_tsdf");
}
