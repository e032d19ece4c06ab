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

// ---------------------------------------------------------------------------- screening
// A point's splat cell is its floor corner c; per cell, mom[27] = sum over its points of
// Fx^a Fy^b Fz^c (index 9a + 3b + c), F the float32 fraction.  Per axis, w(0) = 1 - F and
// w(1) = F, so w(d) w(e) and w(d) are polynomials in F with the coefficients below, and every
// S = sum phi_i phi_j and Phi = sum phi_i of the cell is a fixed combination of its moments.
// mask[node] bit d (d = 4 dx + 2 dy + dz) is set when cell node - d holds points; map[cell] is
// the cell's row in mom.
__device__ __forceinline__ double pair_coef(int d, int e, int k) {
  if (d != e) return k == 0 ? 0.0 : (k == 1 ? 1.0 : -1.0);
  return d ? (k == 2 ? 1.0 : 0.0) : (k == 0 ? 1.0 : (k == 1 ? -2.0 : 1.0));
}

// S[e] = sum_p phi_d(p) phi_e(p) over one cell, for corner d and its 8 corners e (x-major):
// contract the moments over z, then y, then x
__device__ __forceinline__ void cell_row(const double* __restrict__ m, int dx, int dy, int dz,
                                         double (&S)[8]) {
  double tz[2][9];
#pragma unroll
  for (int ez = 0; ez < 2; ++ez)
#pragma unroll
    for (int ab = 0; ab < 9; ++ab) {
      double s = 0.0;
#pragma unroll
      for (int c = 0; c < 3; ++c) s += pair_coef(dz, ez, c) * __ldg(m + ab * 3 + c);
      tz[ez][ab] = s;
    }
#pragma unroll
  for (int ey = 0; ey < 2; ++ey)
#pragma unroll
    for (int ez = 0; ez < 2; ++ez) {
      double ty[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        double s = 0.0;
#pragma unroll
        for (int b = 0; b < 3; ++b) s += pair_coef(dy, ey, b) * tz[ez][a * 3 + b];
        ty[a] = s;
      }
#pragma unroll
      for (int ex = 0; ex < 2; ++ex) {
        double s = 0.0;
#pragma unroll
        for (int a = 0; a < 3; ++a) s += pair_coef(dx, ex, a) * ty[a];
        S[ex * 4 + ey * 2 + ez] = s;
      }
    }
}

// sum_p phi_d(p) over one cell: w(0) = 1 - F, w(1) = F
__device__ __forceinline__ double cell_phi(const double* __restrict__ m, int dx, int dy, int dz) {
  double s = 0.0;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const double w = (dx ? (a ? 1.0 : 0.0) : (a ? -1.0 : 1.0)) *
                         (dy ? (b ? 1.0 : 0.0) : (b ? -1.0 : 1.0)) *
                         (dz ? (c ? 1.0 : 0.0) : (c ? -1.0 : 1.0));
        if (w != 0.0) s += w * __ldg(m + a * 9 + b * 3 + c);
      }
  return s;
}

// splat-cell key of each point: flat floor(p / h) - lo, kPoissonKeyNone when the cell leaves
// 0..N-2 on an axis (its corners would leave the grid)
__global__ void __launch_bounds__(256)
poisson_screen_keys_kernel(const float* __restrict__ pts, int n, float h, int lx, int ly, int lz,
                           int N, long long* __restrict__ keys) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  float fr;
  const int cx = point_axis(pts, j, 0, h, lx, fr), cy = point_axis(pts, j, 1, h, ly, fr),
            cz = point_axis(pts, j, 2, h, lz, fr);
  const bool ok = cx >= 0 && cy >= 0 && cz >= 0 && cx < N - 1 && cy < N - 1 && cz < N - 1;
  keys[j] = ok ? ((long long)cx * N + cy) * N + cz : kPoissonKeyNone;
}

// one thread per cell: the 27 moments of its points (order[start[c]..start[c+1]]) in order
__global__ void __launch_bounds__(128)
poisson_screen_moments_kernel(const float* __restrict__ pts, const int* __restrict__ order,
                              const int* __restrict__ start, int nc, float h, int lx, int ly,
                              int lz, double* __restrict__ mom) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  double m[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) m[k] = 0.0;
  for (int q = __ldg(start + c); q < __ldg(start + c + 1); ++q) {
    const size_t j = (size_t)__ldg(order + q);
    float f[3];
    point_axis(pts, j, 0, h, lx, f[0]);
    point_axis(pts, j, 1, h, ly, f[1]);
    point_axis(pts, j, 2, h, lz, f[2]);
    const double px[3] = {1.0, (double)f[0], (double)f[0] * f[0]};
    const double py[3] = {1.0, (double)f[1], (double)f[1] * f[1]};
    const double pz[3] = {1.0, (double)f[2], (double)f[2] * f[2]};
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const double ab = px[a] * py[b];
#pragma unroll
        for (int k = 0; k < 3; ++k) m[a * 9 + b * 3 + k] += ab * pz[k];
      }
  }
#pragma unroll
  for (int k = 0; k < 27; ++k) mom[(size_t)c * 27 + k] = m[k];
}

// F' = (m + F) / 2 per axis: coefficient of F^k in F'^kk
__device__ __forceinline__ double half_coef(int mbit, int kk, int k) {
  if (kk == 0) return k == 0 ? 1.0 : 0.0;
  if (kk == 1) return k == 1 ? 0.5 : (k == 0 && mbit ? 0.5 : 0.0);
  return k == 2 ? 0.25 : (mbit ? (k == 1 ? 0.5 : 0.25) : 0.0);
}

// one thread per parent cell: the sum over its children m = 0..7 (x-major) of the child
// moments under F' = (m + F) / 2, each transformed over z, then y, then x
__global__ void __launch_bounds__(128)
poisson_screen_coarsen_kernel(const int* __restrict__ cmap, const double* __restrict__ cmom,
                              int nchild, const long long* __restrict__ pkeys, int np,
                              double* __restrict__ pmom) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= np) return;
  const int n = nchild / 2;
  const long long key = __ldg(pkeys + c);
  const int X = (int)(key / ((long long)n * n)), Y = (int)((key / n) % n), Z = (int)(key % n);
  double acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.0;
  for (int m = 0; m < 8; ++m) {
    const int mx = m >> 2, my = (m >> 1) & 1, mz = m & 1;
    const int k = __ldg(cmap + node(2 * X + mx, 2 * Y + my, 2 * Z + mz, nchild));
    if (k < 0) continue;
    const double* M = cmom + (size_t)k * 27;
    double tz[27], ty[27];
#pragma unroll
    for (int ab = 0; ab < 9; ++ab)
#pragma unroll
      for (int kk = 0; kk < 3; ++kk) {
        double s = 0.0;
#pragma unroll
        for (int q = 0; q < 3; ++q) s += half_coef(mz, kk, q) * __ldg(M + ab * 3 + q);
        tz[ab * 3 + kk] = s;
      }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int kk = 0; kk < 3; ++kk)
#pragma unroll
        for (int q3 = 0; q3 < 3; ++q3) {
          double s = 0.0;
#pragma unroll
          for (int q = 0; q < 3; ++q) s += half_coef(my, kk, q) * tz[a * 9 + q * 3 + q3];
          ty[a * 9 + kk * 3 + q3] = s;
        }
#pragma unroll
    for (int kk = 0; kk < 3; ++kk)
#pragma unroll
      for (int r = 0; r < 9; ++r) {
        double s = 0.0;
#pragma unroll
        for (int q = 0; q < 3; ++q) s += half_coef(mx, kk, q) * ty[q * 9 + r];
        acc[kk * 9 + r] += s;
      }
  }
#pragma unroll
  for (int k = 0; k < 27; ++k) pmom[(size_t)c * 27 + k] = acc[k];
}

// b_s = float32(b - gamma_t Phi) at interior nodes of level 0, 0 on the outer layer; part: b_s^2
__global__ void __launch_bounds__(kSumThreads)
poisson_screen_rhs_kernel(const float* __restrict__ b, const unsigned char* __restrict__ mask,
                          const int* __restrict__ map, const double* __restrict__ mom, int N,
                          double gamma_t, float* __restrict__ bs, double* __restrict__ part) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < (size_t)N * N * N) {
    int x, y, z;
    node_xyz(i, N, x, y, z);
    float o = 0.f;
    if (interior(x, y, z, N)) {
      const unsigned bits = __ldg(mask + i);
      double phi = 0.0;
      for (int d = 0; d < 8; ++d) {
        if (!((bits >> d) & 1u)) continue;
        const int dx = d >> 2, dy = (d >> 1) & 1, dz = d & 1;
        const int k = __ldg(map + node(x - dx, y - dy, z - dz, N));
        phi += cell_phi(mom + (size_t)k * 27, dx, dy, dz);
      }
      o = (float)((double)__ldg(b + i) - gamma_t * phi);
    }
    bs[i] = o;
    v = (double)o * o;
  }
  const double s = block_sum(v);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// The 27-point stencil of S at each listed node (a node with a set mask bit): st[k], k = 9 (dx+1)
// + 3 (dy+1) + (dz+1), = sum over the cells d = 0..7 around the node, then their corners t = 0..7,
// of S entries expanded in double; corners at index n drop.  Written as float32 and/or double.
__global__ void __launch_bounds__(128)
poisson_screen_stencil_kernel(const long long* __restrict__ nodes, int ns,
                              const unsigned char* __restrict__ mask, const int* __restrict__ map,
                              const double* __restrict__ mom, int n, float* __restrict__ st32,
                              double* __restrict__ st64) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= ns) return;
  const size_t i = (size_t)__ldg(nodes + s);
  int x, y, z;
  node_xyz(i, n, x, y, z);
  const unsigned bits = __ldg(mask + i);
  double acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.0;
  for (int d = 0; d < 8; ++d) {
    if (!((bits >> d) & 1u)) continue;
    const int dx = d >> 2, dy = (d >> 1) & 1, dz = d & 1;
    const int cx = x - dx, cy = y - dy, cz = z - dz;
    double S[8];
    cell_row(mom + (size_t)__ldg(map + node(cx, cy, cz, n)) * 27, dx, dy, dz, S);
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int tx = t >> 2, ty = (t >> 1) & 1, tz = t & 1;
      if (cx + tx >= n || cy + ty >= n || cz + tz >= n) continue;
      acc[(tx - dx + 1) * 9 + (ty - dy + 1) * 3 + (tz - dz + 1)] += S[t];
    }
  }
#pragma unroll
  for (int k = 0; k < 27; ++k) {
    if (st32) st32[(size_t)s * 27 + k] = (float)acc[k];
    if (st64) st64[(size_t)s * 27 + k] = acc[k];
  }
}

// node_xyz for a power-of-two n <= 1024 (n^3 <= 2^30): shifts, no 64-bit division
__device__ __forceinline__ void node_xyz_pow2(size_t i, int n, int& x, int& y, int& z) {
  const unsigned u = (unsigned)i, s = __ffs(n) - 1, m = (unsigned)n - 1;
  z = (int)(u & m);
  y = (int)((u >> s) & m);
  x = (int)(u >> (2 * s));
}

// sum_{k != 13} st[k] e[node + offset k] (k order), a neighbour at index n (unstored) drops; the
// node is interior, so no offset leaves the grid below
template <typename T, typename S>
__device__ __forceinline__ T stencil_off(const T* e, const S* __restrict__ st, int x, int y, int z,
                                         int n) {
  T off = T(0);
#pragma unroll 1
  for (int k = 0; k < 27; ++k) {
    const int X = x + k / 9 - 1, Y = y + (k / 3) % 3 - 1, Z = z + k % 3 - 1;
    if (k == 13 || X >= n || Y >= n || Z >= n) continue;
    off += (T)__ldg(st + k) * e[node(X, Y, Z, n)];
  }
  return off;
}

// r = b_s - (nbsum(chi) - 6 chi - g S chi) / h^2 at interior nodes of level 0, in double, S the
// double stencil of the surface nodes (srow[node] its row; mask 0: no screening term)
__global__ void __launch_bounds__(kSumThreads)
poisson_screen_residual_kernel(const double* __restrict__ chi, const float* __restrict__ bs,
                               const unsigned char* __restrict__ mask, const int* __restrict__ srow,
                               const double* __restrict__ st, int N, float h, double g,
                               float* __restrict__ r, double* __restrict__ part) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < (size_t)N * N * N) {
    int x, y, z;
    node_xyz_pow2(i, N, x, y, z);
    double ri = 0.0;
    if (interior(x, y, z, N)) {
      const double hh = (double)h * h;
      double a = nbsum(chi, i, N) - 6.0 * chi[i];
      if (__ldg(mask + i)) {
        const double* s = st + (size_t)__ldg(srow + i) * 27;
        a -= g * (__ldg(s + 13) * chi[i] + stencil_off(chi, s, x, y, z, N));
      }
      ri = (double)__ldg(bs + i) - a / hh;
    }
    r[i] = (float)ri;
    v = ri * ri;
  }
  const double s = block_sum(v);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// out = r - (nbsum(e) - 6 e - gl (S e)) / h2 in float32 at the level's interior nodes, 0 elsewhere
__global__ void __launch_bounds__(256)
poisson_screen_mg_residual_kernel(const float* __restrict__ e, const float* __restrict__ r,
                                  const unsigned char* __restrict__ mask,
                                  const int* __restrict__ srow, const float* __restrict__ st,
                                  int n, int level, float h2, float gl, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * n * n) return;
  int x, y, z;
  node_xyz_pow2(i, n, x, y, z);
  float o = 0.f;
  if (level_interior(x, y, z, n, level)) {
    float a = level_nbsum(e, i, x, y, z, n) - 6.f * __ldg(e + i);
    if (__ldg(mask + i)) {
      const float* s = st + (size_t)__ldg(srow + i) * 27;
      a -= gl * (__ldg(s + 13) * __ldg(e + i) + stencil_off(e, s, x, y, z, n));
    }
    o = __ldg(r + i) - a / h2;
  }
  out[i] = o;
}

// neighbour sum without __restrict__: the line smoother reads values its block wrote
__device__ __forceinline__ float plain_nbsum(const float* e, size_t i, int x, int y, int z, int n) {
  const size_t sx = (size_t)n * n, sy = n;
  const float zx = x + 1 < n ? e[i + sx] : 0.f, zy = y + 1 < n ? e[i + sy] : 0.f,
              zz = z + 1 < n ? e[i + 1] : 0.f;
  return ((((e[i - sx] + zx) + e[i - sy]) + zy) + e[i - 1]) + zz;
}

// e = (nbsum - h2 r - gl off) / (6 + gl S_ii), float32; mask 0: (nbsum - h2 r) / 6
__device__ __forceinline__ float screen_update(const float* e, float ri, unsigned bits,
                                               const int* __restrict__ srow,
                                               const float* __restrict__ st, size_t i, int x,
                                               int y, int z, int n, float h2, float gl) {
  const float nb = plain_nbsum(e, i, x, y, z, n);
  if (!bits) return (nb - h2 * ri) / 6.f;
  const float* s = st + (size_t)__ldg(srow + i) * 27;
  return (nb - h2 * ri - gl * stencil_off(e, s, x, y, z, n)) / (6.f + gl * __ldg(s + 13));
}

// Colours 2j and 2j + 1 of an 8-colour sweep (colour = 4 (x&1) + 2 (y&1) + (z&1)): one block per
// z-line (x, y) with 2 (x&1) + (y&1) = j, thread t owning z = 2t and 2t + 1.  The even nodes
// update first; after the barrier the odd nodes read them.  Lines of one (x, y) parity share no
// cell and no neighbour, so this is Gauss-Seidel in the colour order.
__global__ void __launch_bounds__(512)
poisson_screen_smooth_lines_kernel(float* e, const float* __restrict__ r,
                                   const unsigned char* __restrict__ mask,
                                   const int* __restrict__ srow, const float* __restrict__ st,
                                   int n, int level, float h2, float gl, int j) {
  const int m = n / 2;
  const int sm = __ffs(m) - 1;                         // m = n / 2 is a power of two
  const int x = 2 * (int)(blockIdx.x >> sm) + (j >> 1), y = 2 * (int)(blockIdx.x & (m - 1)) + (j & 1);
  const int top = level ? n : n - 1;
  const bool line_in = x > 0 && y > 0 && x < top && y < top;
#pragma unroll
  for (int cz = 0; cz < 2; ++cz) {
    const int z = 2 * (int)threadIdx.x + cz;
    if (line_in && z > 0 && z < top) {
      const size_t i = node(x, y, z, n);
      e[i] = screen_update(e, __ldg(r + i), __ldg(mask + i), srow, st, i, x, y, z, n, h2, gl);
    }
    __syncthreads();
  }
}

// The coarsest grid (n^3 <= 512 nodes) in one block: e = 0, then `sweeps` 8-colour sweeps.
__global__ void __launch_bounds__(512)
poisson_screen_smooth_coarse_kernel(float* __restrict__ e, const float* __restrict__ r,
                                    const unsigned char* __restrict__ mask,
                                    const int* __restrict__ srow, const float* __restrict__ st,
                                    int n, int level, float h2, float gl, int sweeps) {
  __shared__ float se[512];
  const int i = threadIdx.x, nn = n * n * n;
  int x = 0, y = 0, z = 0;
  if (i < nn) node_xyz(i, n, x, y, z);
  const bool in = i < nn && level_interior(x, y, z, n, level);
  const float ri = in ? r[i] : 0.f;
  const unsigned bits = in ? mask[i] : 0u;
  const int mine = 4 * (x & 1) + 2 * (y & 1) + (z & 1);
  if (i < nn) se[i] = 0.f;
  __syncthreads();
  for (int s = 0; s < sweeps; ++s)
    for (int colour = 0; colour < 8; ++colour) {
      if (in && mine == colour) se[i] = screen_update(se, ri, bits, srow, st, i, x, y, z, n, h2, gl);
      __syncthreads();
    }
  if (i < nn) e[i] = se[i];
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

extern "C" int casmvs_poisson_screen_keys(const float* points, int n, float h, int lo_x, int lo_y,
                                          int lo_z, int N, long long* keys, void* stream) {
  CASMVS_REQUIRE(n >= 0, "poisson_screen_keys: n < 0");
  CASMVS_REQUIRE(h > 0.f, "poisson_screen_keys: h must be > 0");
  POISSON_GRID("poisson_screen_keys", N);
  if (n == 0) return 0;
  CASMVS_REQUIRE(points && keys, "poisson_screen_keys: null pointer");
  poisson_screen_keys_kernel<<<pblocks(n), 256, 0, as_stream(stream)>>>(points, n, h, lo_x, lo_y,
                                                                        lo_z, N, keys);
  return after_launch("poisson_screen_keys");
}

extern "C" int casmvs_poisson_screen_moments(const float* points, const int* order,
                                             const int* cell_start, int n_cells, float h, int lo_x,
                                             int lo_y, int lo_z, double* moments, void* stream) {
  CASMVS_REQUIRE(n_cells >= 0, "poisson_screen_moments: n_cells < 0");
  CASMVS_REQUIRE(h > 0.f, "poisson_screen_moments: h must be > 0");
  if (n_cells == 0) return 0;
  CASMVS_REQUIRE(points && order && cell_start && moments, "poisson_screen_moments: null pointer");
  poisson_screen_moments_kernel<<<(n_cells + 127) / 128, 128, 0, as_stream(stream)>>>(
      points, order, cell_start, n_cells, h, lo_x, lo_y, lo_z, moments);
  return after_launch("poisson_screen_moments");
}

extern "C" int casmvs_poisson_screen_coarsen(const int* child_map, const double* child_moments,
                                             int n_child, const long long* parent_keys,
                                             int n_parents, double* parent_moments, void* stream) {
  POISSON_GRID("poisson_screen_coarsen", n_child);
  CASMVS_REQUIRE(n_child >= 16, "poisson_screen_coarsen: the child grid needs >= 16 nodes per axis");
  CASMVS_REQUIRE(n_parents >= 0, "poisson_screen_coarsen: n_parents < 0");
  if (n_parents == 0) return 0;
  CASMVS_REQUIRE(child_map && child_moments && parent_keys && parent_moments,
                 "poisson_screen_coarsen: null pointer");
  poisson_screen_coarsen_kernel<<<(n_parents + 127) / 128, 128, 0, as_stream(stream)>>>(
      child_map, child_moments, n_child, parent_keys, n_parents, parent_moments);
  return after_launch("poisson_screen_coarsen");
}

extern "C" int casmvs_poisson_screen_rhs(const float* b, const unsigned char* mask, const int* map,
                                         const double* moments, int N, double gamma_t, float* b_s,
                                         double* workspace, double* bb, void* stream) {
  POISSON_GRID("poisson_screen_rhs", N);
  CASMVS_REQUIRE(b && mask && map && moments && b_s && workspace && bb,
                 "poisson_screen_rhs: null pointer");
  const unsigned nblk = pblocks((size_t)N * N * N);
  poisson_screen_rhs_kernel<<<nblk, kSumThreads, 0, as_stream(stream)>>>(b, mask, map, moments, N,
                                                                         gamma_t, b_s, workspace);
  const int rc = after_launch("poisson_screen_rhs");
  return rc ? rc : finish_sum(workspace, (int)nblk, bb, as_stream(stream), "poisson_screen_rhs");
}

extern "C" int casmvs_poisson_screen_stencil(const long long* nodes, int n_nodes,
                                             const unsigned char* mask, const int* map,
                                             const double* moments, int n, float* stencil32,
                                             double* stencil64, void* stream) {
  POISSON_GRID("poisson_screen_stencil", n);
  CASMVS_REQUIRE(n_nodes >= 0, "poisson_screen_stencil: n_nodes < 0");
  if (n_nodes == 0) return 0;
  CASMVS_REQUIRE(nodes && mask && map && moments && (stencil32 || stencil64),
                 "poisson_screen_stencil: null pointer");
  poisson_screen_stencil_kernel<<<(n_nodes + 127) / 128, 128, 0, as_stream(stream)>>>(
      nodes, n_nodes, mask, map, moments, n, stencil32, stencil64);
  return after_launch("poisson_screen_stencil");
}

extern "C" int casmvs_poisson_screen_residual(const double* chi, const float* b_s,
                                              const unsigned char* mask, const int* srow,
                                              const double* stencil, int N, float h, double g,
                                              float* r, double* workspace, double* rr,
                                              void* stream) {
  POISSON_GRID("poisson_screen_residual", N);
  CASMVS_REQUIRE(h > 0.f && g >= 0.0, "poisson_screen_residual: need h > 0 and g >= 0");
  CASMVS_REQUIRE(chi && b_s && mask && srow && stencil && r && workspace && rr,
                 "poisson_screen_residual: null pointer");
  const unsigned nblk = pblocks((size_t)N * N * N);
  poisson_screen_residual_kernel<<<nblk, kSumThreads, 0, as_stream(stream)>>>(
      chi, b_s, mask, srow, stencil, N, h, g, r, workspace);
  const int rc = after_launch("poisson_screen_residual");
  return rc ? rc : finish_sum(workspace, (int)nblk, rr, as_stream(stream), "poisson_screen_residual");
}

extern "C" int casmvs_poisson_screen_mg_residual(const float* e, const float* r,
                                                 const unsigned char* mask, const int* srow,
                                                 const float* stencil, int n, int level, float h,
                                                 double g, float* out, void* stream) {
  POISSON_GRID("poisson_screen_mg_residual", n);
  CASMVS_REQUIRE(level >= 0, "poisson_screen_mg_residual: level < 0");
  CASMVS_REQUIRE(h > 0.f && g >= 0.0, "poisson_screen_mg_residual: need h > 0 and g >= 0");
  CASMVS_REQUIRE(e && r && mask && srow && stencil && out, "poisson_screen_mg_residual: null pointer");
  poisson_screen_mg_residual_kernel<<<pblocks((size_t)n * n * n), 256, 0, as_stream(stream)>>>(
      e, r, mask, srow, stencil, n, level, h * h, (float)ldexp(g, -level), out);
  return after_launch("poisson_screen_mg_residual");
}

extern "C" int casmvs_poisson_screen_smooth(float* e, const float* r, const unsigned char* mask,
                                            const int* srow, const float* stencil, int n, int level,
                                            float h, double g, int sweeps, int zero_first,
                                            void* stream) {
  POISSON_GRID("poisson_screen_smooth", n);
  CASMVS_REQUIRE(level >= 0, "poisson_screen_smooth: level < 0");
  CASMVS_REQUIRE(h > 0.f && g >= 0.0 && sweeps >= 0,
                 "poisson_screen_smooth: need h > 0, g >= 0 and sweeps >= 0");
  CASMVS_REQUIRE(e && r && mask && srow && stencil, "poisson_screen_smooth: null pointer");
  const float h2 = h * h;
  const float gl = (float)ldexp(g, -level);         // gamma_l h_l^2 = (gamma / 8^l) (2^l h)^2
  const size_t nn = (size_t)n * n * n;
  cudaStream_t st = as_stream(stream);
  if (zero_first && nn <= 512) {
    poisson_screen_smooth_coarse_kernel<<<1, 512, 0, st>>>(e, r, mask, srow, stencil, n, level, h2,
                                                           gl, sweeps);
    return after_launch("poisson_screen_smooth");
  }
  if (zero_first) {
    cudaError_t err = cudaMemsetAsync(e, 0, nn * sizeof(float), st);
    CASMVS_REQUIRE(err == cudaSuccess, "poisson_screen_smooth: memset failed: %s",
                   cudaGetErrorString(err));
  }
  const unsigned lines = (unsigned)((n / 2) * (n / 2));
  for (int s = 0; s < sweeps; ++s)
    for (int j = 0; j < 4; ++j) {
      poisson_screen_smooth_lines_kernel<<<lines, n / 2, 0, st>>>(e, r, mask, srow, stencil, n,
                                                                  level, h2, gl, j);
      const int rc = after_launch("poisson_screen_smooth");
      if (rc) return rc;
    }
  return 0;
}
