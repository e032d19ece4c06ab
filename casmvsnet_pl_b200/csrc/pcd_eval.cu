// DTU point-cloud scoring on the GPU: grid binning, 0.2 mm thinning and capped nearest-neighbour
// distances.  Restates the reference's MATLAB scorer (paths relative to the reference root):
//   reducePts_haa.m                greedy thinning in a random visiting order
//   MaxDistCP.m                    nearest-neighbour distance inside 60 mm blocks, 60 elsewhere
//   PointCompareMain.m:7,20-24     dst = 0.2 mm, MaxDist = 60 mm, Ddata / Dstl
// The masks and statistics (PointCompareMain.m:32-53, ComputeStat_web.m) are torch ops in
// casmvsnet_pl_b200/dtu_eval.py; the sort and run-length scan that turn cell keys into cells are
// torch plumbing as well.
//
// Thinning.  Visiting points in rank order and keeping every point no kept point lies within
// dst of gives the lexicographically-first maximal independent set (LFMIS) of the "<= dst" graph.
// It is computed in parallel rounds: an undecided point joins when no undecided-or-kept neighbour
// has a lower rank (pcd_thin_join), then every undecided neighbour of a kept point is removed
// (pcd_thin_remove).  A point joins exactly when all its lower-ranked neighbours are removed,
// which is the sequential rule, so the set does not depend on thread scheduling.  Both kernels
// only move a point 0 -> 1 or 0 -> 2 and the readers of a racing write take the same decision
// from either value, so the rounds need no atomics beyond the undecided counter.
//
// Nearest neighbour.  Targets are binned into cells of h mm grouped in super cells of 8^3 cells;
// keys sort super-major, so a super cell's occupied cells are one contiguous run of the cell
// list and a dense table (super_begin) gives that run.  A query walks Chebyshev rings of super
// cells outwards, skips empty supers and supers / cells whose box is farther than the best
// distance so far (initially the 60 mm cap), and stops once the next ring cannot be closer.  A
// query far from every target therefore visits O((cap / 8h)^2) super cells per ring, not the
// (cap / h)^3 cells of a 60 mm ball.
#include "common.cuh"

namespace casmvs {

constexpr int kNbr = 27;
constexpr int64_t kOutsideKey = INT64_MAX;

// ---------------------------------------------------------------------------------- binning
// Plain layout (sub == 1): key = (ix * gy + iy) * gz + iz.
// Super layout (sub == 8): key = ((sx * SY + sy) * SZ + sz) << 9 | lx << 6 | ly << 3 | lz with
// s = i >> 3, l = i & 7 and S = ceil(g / 8).  Points outside [0, g) get kOutsideKey.
__global__ void __launch_bounds__(256)
pcd_cell_keys_kernel(const float* __restrict__ pts, int n, double ox, double oy, double oz,
                     double cell, int gx, int gy, int gz, int sub, int64_t* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double fx = floor(((double)__ldg(pts + 3 * (size_t)i) - ox) / cell);
  const double fy = floor(((double)__ldg(pts + 3 * (size_t)i + 1) - oy) / cell);
  const double fz = floor(((double)__ldg(pts + 3 * (size_t)i + 2) - oz) / cell);
  // NaN fails every comparison and lands outside as well
  if (!(fx >= 0.0 && fx < gx && fy >= 0.0 && fy < gy && fz >= 0.0 && fz < gz)) {
    keys[i] = kOutsideKey;
    return;
  }
  const int64_t ix = (int64_t)fx, iy = (int64_t)fy, iz = (int64_t)fz;
  if (sub == 1) {
    keys[i] = (ix * gy + iy) * gz + iz;
  } else {
    const int64_t SY = (gy + 7) >> 3, SZ = (gz + 7) >> 3;
    const int64_t s = ((ix >> 3) * SY + (iy >> 3)) * SZ + (iz >> 3);
    keys[i] = (s << 9) | ((ix & 7) << 6) | ((iy & 7) << 3) | (iz & 7);
  }
}

// ---------------------------------------------------------------------------------- thinning
// |p - q| <= dst on float32 coordinates, evaluated in double in a fixed operation order
// ((dx*dx + dy*dy) + dz*dz <= dst*dst, no contraction) so that a float64 oracle that writes the
// same expression keeps exactly the same points.
__device__ __forceinline__ bool within_dst(const float* __restrict__ pts, int p, double px,
                                          double py, double pz, double dst2) {
  const double dx = __dsub_rn((double)pts[3 * (size_t)p], px);
  const double dy = __dsub_rn((double)pts[3 * (size_t)p + 1], py);
  const double dz = __dsub_rn((double)pts[3 * (size_t)p + 2], pz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) <= dst2;
}

// One thread per occupied cell: the 27 neighbour cells (index into the cell list or -1) by
// binary search of the sorted unique keys, and the cell index of each of its points.
__global__ void __launch_bounds__(256)
pcd_thin_prepare_kernel(const int64_t* __restrict__ cell_keys, const int* __restrict__ cell_start,
                        int ncells, int gx, int gy, int gz, int* __restrict__ nbr,
                        int* __restrict__ cell_of) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncells) return;
  const int64_t k = __ldg(cell_keys + c);
  const int64_t ix = k / ((int64_t)gy * gz), rem = k - ix * ((int64_t)gy * gz);
  const int64_t iy = rem / gz, iz = rem - iy * gz;
  int j = 0;
  for (int dx = -1; dx <= 1; ++dx)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dz = -1; dz <= 1; ++dz, ++j) {
        const int64_t x = ix + dx, y = iy + dy, z = iz + dz;
        int found = -1;
        if (x >= 0 && x < gx && y >= 0 && y < gy && z >= 0 && z < gz) {
          const int64_t want = (x * gy + y) * gz + z;
          int lo = 0, hi = ncells;                      // first key >= want
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(cell_keys + mid) < want) lo = mid + 1; else hi = mid;
          }
          if (lo < ncells && __ldg(cell_keys + lo) == want) found = lo;
        }
        nbr[(size_t)c * kNbr + j] = found;
      }
  for (int p = __ldg(cell_start + c), e = __ldg(cell_start + c + 1); p < e; ++p) cell_of[p] = c;
}

// state: 0 undecided, 1 kept, 2 removed.  Racing writes only move other points 0 -> 1, and the
// join test reads "not removed" from either value: plain (non-__ldg) loads of `state`.
__global__ void __launch_bounds__(256)
pcd_thin_join_kernel(const float* __restrict__ pts, const int* __restrict__ rank,
                     const int* __restrict__ cell_start, const int* __restrict__ nbr,
                     const int* __restrict__ cell_of, int n, double dst2, unsigned char* state) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n || state[p] != 0) return;
  const int rp = __ldg(rank + p);
  const double px = (double)__ldg(pts + 3 * (size_t)p), py = (double)__ldg(pts + 3 * (size_t)p + 1),
               pz = (double)__ldg(pts + 3 * (size_t)p + 2);
  const int* nb = nbr + (size_t)__ldg(cell_of + p) * kNbr;
  for (int j = 0; j < kNbr; ++j) {
    const int c = __ldg(nb + j);
    if (c < 0) continue;
    for (int q = __ldg(cell_start + c), e = __ldg(cell_start + c + 1); q < e; ++q) {
      if (__ldg(rank + q) < rp && state[q] != 2 && within_dst(pts, q, px, py, pz, dst2)) return;
    }
  }
  state[p] = 1;
}

// Removes the undecided neighbours of kept points and counts the points still undecided.  Racing
// writes only move other points 0 -> 2, and the test reads "kept" from neither value.
__global__ void __launch_bounds__(256)
pcd_thin_remove_kernel(const float* __restrict__ pts, const int* __restrict__ cell_start,
                       const int* __restrict__ nbr, const int* __restrict__ cell_of, int n,
                       double dst2, unsigned char* state, int* __restrict__ undecided) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  bool left = false;
  if (p < n && state[p] == 0) {
    const double px = (double)__ldg(pts + 3 * (size_t)p),
                 py = (double)__ldg(pts + 3 * (size_t)p + 1),
                 pz = (double)__ldg(pts + 3 * (size_t)p + 2);
    const int* nb = nbr + (size_t)__ldg(cell_of + p) * kNbr;
    bool hit = false;
    for (int j = 0; j < kNbr && !hit; ++j) {
      const int c = __ldg(nb + j);
      if (c < 0) continue;
      for (int q = __ldg(cell_start + c), e = __ldg(cell_start + c + 1); q < e; ++q) {
        if (state[q] == 1 && within_dst(pts, q, px, py, pz, dst2)) { hit = true; break; }
      }
    }
    if (hit) state[p] = 2; else left = true;
  }
  const unsigned m = __ballot_sync(0xffffffffu, left);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(undecided, __popc(m));
}

// ---------------------------------------------------------------------------------- capped NN
struct NNGrid {
  double org[3];      // corner of fine cell (0,0,0)
  double h;           // fine cell edge
  double hs;          // super cell edge = 8h
  int S[3];           // super dims
  double lo[3], hi[3];  // query block grid: lo <= q < hi on every axis (MaxDistCP.m:5-18)
  double cap, cap2;
};

// squared distance from q to the box [b, b + e]^3, boxes widened by 1e-6 mm so that a point
// binned into a cell by a rounded floor() is never pruned with it
__device__ __forceinline__ double box_d2(const double q[3], double bx, double by, double bz,
                                         double e) {
  const double b[3] = {bx - 1e-6, by - 1e-6, bz - 1e-6};
  double d2 = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double lo = b[a], hi = b[a] + e + 2e-6;
    const double d = q[a] < lo ? lo - q[a] : (q[a] > hi ? q[a] - hi : 0.0);
    d2 += d * d;
  }
  return d2;
}

// kIndex == false is the DTU search (casmvs_pcd_capped_nn).  kIndex == true also returns the
// original index of the nearest target (tgt_index maps the key-sorted targets back): it evaluates
// the distance with explicit round-to-nearest intrinsics in the same order, breaks an exact tie
// towards the lower original index and prunes only boxes strictly farther than the best distance,
// so that a tied target in another cell is still visited.
template <bool kIndex>
__device__ __forceinline__ void scan_super(const NNGrid& G, const double q[3], int sx, int sy,
                                           int sz, const int* __restrict__ super_begin,
                                           const int64_t* __restrict__ cell_keys,
                                           const int* __restrict__ cell_start,
                                           const float* __restrict__ tgt,
                                           const int64_t* __restrict__ tgt_index, double& best2,
                                           int64_t& best_i) {
  const int s = (sx * G.S[1] + sy) * G.S[2] + sz;
  const int c0 = __ldg(super_begin + s), c1 = __ldg(super_begin + s + 1);
  if (c0 == c1) return;
  const double bx = G.org[0] + sx * G.hs, by = G.org[1] + sy * G.hs, bz = G.org[2] + sz * G.hs;
  const double sd2 = box_d2(q, bx, by, bz, G.hs);
  if (kIndex ? sd2 > best2 : sd2 >= best2) return;
  for (int c = c0; c < c1; ++c) {
    const int l = (int)(__ldg(cell_keys + c) & 511);
    const double cd2 = box_d2(q, bx + (l >> 6) * G.h, by + ((l >> 3) & 7) * G.h, bz + (l & 7) * G.h, G.h);
    if (kIndex ? cd2 > best2 : cd2 >= best2) continue;
    for (int t = __ldg(cell_start + c), e = __ldg(cell_start + c + 1); t < e; ++t) {
      if constexpr (kIndex) {
        const double dx = __dsub_rn((double)__ldg(tgt + 3 * (size_t)t), q[0]);
        const double dy = __dsub_rn((double)__ldg(tgt + 3 * (size_t)t + 1), q[1]);
        const double dz = __dsub_rn((double)__ldg(tgt + 3 * (size_t)t + 2), q[2]);
        const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
        if (d2 <= best2) {
          const int64_t id = __ldg(tgt_index + t);
          if (d2 < best2 || id < best_i) {
            best2 = d2;
            best_i = id;
          }
        }
      } else {
        const double dx = (double)__ldg(tgt + 3 * (size_t)t) - q[0];
        const double dy = (double)__ldg(tgt + 3 * (size_t)t + 1) - q[1];
        const double dz = (double)__ldg(tgt + 3 * (size_t)t + 2) - q[2];
        best2 = fmin(best2, dx * dx + dy * dy + dz * dz);
      }
    }
  }
}

template <bool kIndex>
__global__ void __launch_bounds__(128, kIndex ? 8 : 0)
pcd_capped_nn_kernel(const __grid_constant__ NNGrid G, const float* __restrict__ qry, int nq,
                     const float* __restrict__ tgt, const int64_t* __restrict__ cell_keys,
                     const int* __restrict__ cell_start, const int* __restrict__ super_begin,
                     const int64_t* __restrict__ tgt_index, double* __restrict__ dist,
                     int64_t* __restrict__ index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const double q[3] = {(double)__ldg(qry + 3 * (size_t)i), (double)__ldg(qry + 3 * (size_t)i + 1),
                       (double)__ldg(qry + 3 * (size_t)i + 2)};
  bool inside = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) inside = inside && q[a] >= G.lo[a] && q[a] < G.hi[a];
  if (!inside || super_begin == nullptr) {       // outside every block, or no target at all
    dist[i] = G.cap;
    if (kIndex) index[i] = -1;
    return;
  }
  // the target grid spans the block grid widened by the cap, so an inside query is in it
  int c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    c[a] = min(max((int)floor((q[a] - G.org[a]) / G.hs), 0), G.S[a] - 1);
  double best2 = G.cap2;
  int64_t best_i = INT64_MAX;
  const int rmax = max(G.S[0], max(G.S[1], G.S[2]));
  for (int R = 0; R <= rmax; ++R) {
    // every cell of ring R is at least (R - 1) super edges away along one axis
    const double lb = (R - 1) * G.hs - 1e-6;
    if (R >= 2 && (kIndex ? lb * lb > best2 : lb * lb >= best2)) break;
    const int x0 = max(c[0] - R, 0), x1 = min(c[0] + R, G.S[0] - 1);
    const int y0 = max(c[1] - R, 0), y1 = min(c[1] + R, G.S[1] - 1);
    for (int x = x0; x <= x1; ++x) {
      const bool xface = x == c[0] - R || x == c[0] + R;
      for (int y = y0; y <= y1; ++y) {
        const bool face = xface || y == c[1] - R || y == c[1] + R;
        if (face) {
          const int z0 = max(c[2] - R, 0), z1 = min(c[2] + R, G.S[2] - 1);
          for (int z = z0; z <= z1; ++z)
            scan_super<kIndex>(G, q, x, y, z, super_begin, cell_keys, cell_start, tgt, tgt_index,
                               best2, best_i);
        } else {
          if (c[2] - R >= 0)
            scan_super<kIndex>(G, q, x, y, c[2] - R, super_begin, cell_keys, cell_start, tgt,
                               tgt_index, best2, best_i);
          if (R > 0 && c[2] + R < G.S[2])
            scan_super<kIndex>(G, q, x, y, c[2] + R, super_begin, cell_keys, cell_start, tgt,
                               tgt_index, best2, best_i);
        }
      }
    }
  }
  dist[i] = best2 < G.cap2 ? sqrt(best2) : G.cap;
  if (kIndex) index[i] = best2 < G.cap2 ? best_i : -1;
}

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_pcd_cell_keys(const float* points, int n, double ox, double oy, double oz,
                                    double cell, int gx, int gy, int gz, int sub, int64_t* keys,
                                    void* stream) {
  CASMVS_REQUIRE(n >= 0, "pcd_cell_keys: n < 0");
  CASMVS_REQUIRE(sub == 1 || sub == 8, "pcd_cell_keys: sub must be 1 or 8");
  CASMVS_REQUIRE(cell > 0.0, "pcd_cell_keys: cell size must be > 0");
  CASMVS_REQUIRE(gx > 0 && gy > 0 && gz > 0 && gx < (1 << 20) && gy < (1 << 20) && gz < (1 << 20),
                 "pcd_cell_keys: grid dims must lie in [1, 2^20)");
  CASMVS_REQUIRE(n == 0 || (points && keys), "pcd_cell_keys: null pointer");
  if (n == 0) return 0;
  pcd_cell_keys_kernel<<<(n + 255) / 256, 256, 0, as_stream(stream)>>>(points, n, ox, oy, oz, cell,
                                                                        gx, gy, gz, sub, keys);
  return after_launch("pcd_cell_keys");
}

extern "C" size_t casmvs_pcd_thin_workspace_bytes(int n, int ncells) {
  if (n < 0 || ncells < 0) return 0;
  const size_t nbr = ((size_t)ncells * kNbr * sizeof(int) + 255) & ~(size_t)255;
  return nbr + (size_t)n * sizeof(int);
}

extern "C" int casmvs_pcd_thin_prepare(const int64_t* cell_keys, const int* cell_start, int n,
                                       int ncells, int gx, int gy, int gz, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  CASMVS_REQUIRE(n >= 0 && ncells >= 0 && ncells <= n, "pcd_thin_prepare: bad sizes");
  CASMVS_REQUIRE(gx > 0 && gy > 0 && gz > 0, "pcd_thin_prepare: bad grid dims");
  CASMVS_REQUIRE(workspace_bytes >= casmvs_pcd_thin_workspace_bytes(n, ncells),
                 "pcd_thin_prepare: workspace too small (%zu < %zu bytes)", workspace_bytes,
                 casmvs_pcd_thin_workspace_bytes(n, ncells));
  CASMVS_REQUIRE(ncells == 0 || (cell_keys && cell_start && workspace), "pcd_thin_prepare: null pointer");
  if (ncells == 0) return 0;
  int* nbr = static_cast<int*>(workspace);
  int* cell_of = reinterpret_cast<int*>(static_cast<char*>(workspace) +
                                        casmvs_pcd_thin_workspace_bytes(0, ncells));
  pcd_thin_prepare_kernel<<<(ncells + 255) / 256, 256, 0, as_stream(stream)>>>(
      cell_keys, cell_start, ncells, gx, gy, gz, nbr, cell_of);
  return after_launch("pcd_thin_prepare");
}

extern "C" int casmvs_pcd_thin_round(const float* points, const int* rank, const int* cell_start,
                                     int n, int ncells, double dst, unsigned char* state,
                                     int* undecided, const void* workspace,
                                     size_t workspace_bytes, void* stream) {
  CASMVS_REQUIRE(n >= 0 && ncells >= 0 && ncells <= n, "pcd_thin_round: bad sizes");
  CASMVS_REQUIRE(dst >= 0.0, "pcd_thin_round: dst must be >= 0");
  CASMVS_REQUIRE(undecided, "pcd_thin_round: null pointer");
  CASMVS_REQUIRE(workspace_bytes >= casmvs_pcd_thin_workspace_bytes(n, ncells),
                 "pcd_thin_round: workspace too small (%zu < %zu bytes)", workspace_bytes,
                 casmvs_pcd_thin_workspace_bytes(n, ncells));
  CASMVS_REQUIRE(n == 0 || (points && rank && cell_start && state && workspace),
                 "pcd_thin_round: null pointer");
  cudaStream_t st = as_stream(stream);
  if (cudaMemsetAsync(undecided, 0, sizeof(int), st) != cudaSuccess) {
    set_error("pcd_thin_round: cudaMemsetAsync failed");
    return -2;
  }
  if (n == 0) return 0;
  const int* nbr = static_cast<const int*>(workspace);
  const int* cell_of = reinterpret_cast<const int*>(static_cast<const char*>(workspace) +
                                                    casmvs_pcd_thin_workspace_bytes(0, ncells));
  const double dst2 = dst * dst;
  pcd_thin_join_kernel<<<(n + 255) / 256, 256, 0, st>>>(points, rank, cell_start, nbr, cell_of, n,
                                                        dst2, state);
  if (int rc = after_launch("pcd_thin_join")) return rc;
  pcd_thin_remove_kernel<<<(n + 255) / 256, 256, 0, st>>>(points, cell_start, nbr, cell_of, n,
                                                          dst2, state, undecided);
  return after_launch("pcd_thin_remove");
}

static int capped_nn_launch(const char* what, const float* queries, int nq, const float* targets,
                            const int64_t* cell_keys, const int* cell_start, int ncells,
                            const int* super_begin, const double* origin3, double h,
                            const int* super_dims3, const double* box_lo3, const double* box_hi3,
                            double cap, const int64_t* target_index, double* dist, int64_t* index,
                            void* stream) {
  CASMVS_REQUIRE(nq >= 0 && ncells >= 0, "%s: bad sizes", what);
  CASMVS_REQUIRE(origin3 && super_dims3 && box_lo3 && box_hi3, "%s: null host array", what);
  CASMVS_REQUIRE(h > 0.0 && cap > 0.0, "%s: h and cap must be > 0", what);
  CASMVS_REQUIRE(nq == 0 || (queries && dist), "%s: null pointer", what);
  CASMVS_REQUIRE(ncells == 0 || (targets && cell_keys && cell_start && super_begin),
                 "%s: null target pointer", what);
  NNGrid G;
  size_t nsuper = 1;
  for (int a = 0; a < 3; ++a) {
    CASMVS_REQUIRE(super_dims3[a] > 0 && super_dims3[a] < (1 << 17), "%s: bad super dims", what);
    nsuper *= (size_t)super_dims3[a];
    G.org[a] = origin3[a];
    G.S[a] = super_dims3[a];
    G.lo[a] = box_lo3[a];
    G.hi[a] = box_hi3[a];
  }
  CASMVS_REQUIRE(nsuper < (1u << 31), "%s: too many super cells", what);
  G.h = h;
  G.hs = 8.0 * h;
  G.cap = cap;
  G.cap2 = cap * cap;
  if (nq == 0) return 0;
  const int* sb = ncells ? super_begin : nullptr;
  if (index) {
    pcd_capped_nn_kernel<true><<<(nq + 127) / 128, 128, 0, as_stream(stream)>>>(
        G, queries, nq, targets, cell_keys, cell_start, sb, target_index, dist, index);
  } else {
    pcd_capped_nn_kernel<false><<<(nq + 127) / 128, 128, 0, as_stream(stream)>>>(
        G, queries, nq, targets, cell_keys, cell_start, sb, nullptr, dist, nullptr);
  }
  return after_launch(what);
}

extern "C" int casmvs_pcd_capped_nn(const float* queries, int nq, const float* targets,
                                    const int64_t* cell_keys, const int* cell_start, int ncells,
                                    const int* super_begin, const double* origin3, double h,
                                    const int* super_dims3, const double* box_lo3,
                                    const double* box_hi3, double cap, double* dist,
                                    void* stream) {
  return capped_nn_launch("pcd_capped_nn", queries, nq, targets, cell_keys, cell_start, ncells,
                          super_begin, origin3, h, super_dims3, box_lo3, box_hi3, cap, nullptr,
                          dist, nullptr, stream);
}

extern "C" int casmvs_pcd_capped_nn_index(const float* queries, int nq, const float* targets,
                                          const int64_t* cell_keys, const int* cell_start,
                                          int ncells, const int* super_begin,
                                          const double* origin3, double h, const int* super_dims3,
                                          const double* box_lo3, const double* box_hi3, double cap,
                                          const int64_t* target_index, double* dist,
                                          int64_t* index, void* stream) {
  CASMVS_REQUIRE(nq == 0 || index, "pcd_capped_nn_index: null index pointer");
  CASMVS_REQUIRE(ncells == 0 || target_index, "pcd_capped_nn_index: null target_index pointer");
  return capped_nn_launch("pcd_capped_nn_index", queries, nq, targets, cell_keys, cell_start,
                          ncells, super_begin, origin3, h, super_dims3, box_lo3, box_hi3, cap,
                          target_index, dist, index, stream);
}
