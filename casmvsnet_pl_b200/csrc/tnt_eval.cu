// Tanks and Temples scoring on the GPU (casmvsnet_pl_b200/tnt_eval.py): the per-point steps of the
// training-set evaluation.  The nearest-neighbour search is pcd_eval.cu's capped grid search
// (casmvs_pcd_capped_nn_index); sorting cell keys, the run-length scan that turns them into
// voxels, the block-offset scan of the compaction and the score histograms are torch plumbing.
//
// Every float operation whose result a float64 oracle (oracle/tnt_eval_oracle.py) restates bit for
// bit is an explicit round-to-nearest intrinsic in the order the header states, so that nvcc
// cannot contract it into an FMA.
//
// Transform + crop.  One thread per point: p' = float32(T p) in double, then Open3D's
// CropInPolygon test on p' (axis bounds, then an even-odd count of the polygon nodes below p'.v).
// A CTA counts its kept points (__syncthreads_count); after an exclusive scan of those counts the
// compaction pass writes each kept point at its CTA's offset plus its rank inside the CTA, so the
// output keeps input order without atomics.
//
// Voxel mean.  One thread per occupied voxel sums its points in input order (a stable key sort
// keeps it) in double and rounds the mean to float32.
//
// ICP moments.  A fixed grid (a function of n alone) of grid-stride threads accumulates 18 double
// sums per thread in index order, CTAs reduce them in a fixed tree and one CTA adds the CTA sums
// in order: the same bits on every run, with no float atomics.
#include "common.cuh"

namespace casmvs {

constexpr int kCropThreads = 256;
constexpr int kMomThreads = 256;
constexpr int kMomMaxBlocks = 1024;
constexpr int kMoments = 18;

struct CropParams {
  double T[12];         // rows 0..2 of the 4x4 transform, row-major
  int transform;        // 0: points are used as they are
  int crop;             // 0: every point is kept (mask and counts are not written)
  int axis;             // orthogonal axis; the polygon's plane axes (u, v) follow from it
  double amin, amax;
  int m;                // polygon vertices (u, v) pairs in `poly`
};

__device__ __forceinline__ float xf_row(const double* r, double x, double y, double z) {
  return __double2float_rn(
      __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], x), __dmul_rn(r[1], y)), __dmul_rn(r[2], z)), r[3]));
}

__device__ __forceinline__ bool in_polygon(const CropParams& P, const double* __restrict__ poly,
                                           double x, double y, double z) {
  const double pa = P.axis == 0 ? x : (P.axis == 1 ? y : z);
  if (pa < P.amin || pa > P.amax) return false;
  const double pu = P.axis == 0 ? y : x, pv = P.axis == 2 ? y : z;
  int below = 0;
  for (int i = 0; i < P.m; ++i) {
    const int j = i + 1 == P.m ? 0 : i + 1;
    const double iu = __ldg(poly + 2 * i), iv = __ldg(poly + 2 * i + 1);
    const double ju = __ldg(poly + 2 * j), jv = __ldg(poly + 2 * j + 1);
    if ((iu < pu && ju >= pu) || (ju < pu && iu >= pu)) {
      const double node =
          __dadd_rn(iv, __dmul_rn(__ddiv_rn(__dsub_rn(pu, iu), __dsub_rn(ju, iu)), __dsub_rn(jv, iv)));
      below += node < pv;        // lower_bound on the sorted nodes = the count of nodes < p.v
    }
  }
  return below & 1;
}

__global__ void __launch_bounds__(kCropThreads)
tnt_transform_crop_kernel(const float* __restrict__ pts, int n, const __grid_constant__ CropParams P,
                          const double* __restrict__ poly, float* __restrict__ out,
                          unsigned char* __restrict__ mask, int* __restrict__ block_counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool keep = false;
  if (i < n) {
    float f[3] = {__ldg(pts + 3 * (size_t)i), __ldg(pts + 3 * (size_t)i + 1),
                  __ldg(pts + 3 * (size_t)i + 2)};
    if (P.transform) {
      const double x = f[0], y = f[1], z = f[2];
      f[0] = xf_row(P.T, x, y, z);
      f[1] = xf_row(P.T + 4, x, y, z);
      f[2] = xf_row(P.T + 8, x, y, z);
    }
    out[3 * (size_t)i] = f[0];
    out[3 * (size_t)i + 1] = f[1];
    out[3 * (size_t)i + 2] = f[2];
    if (P.crop) {
      keep = in_polygon(P, poly, f[0], f[1], f[2]);
      mask[i] = keep;
    }
  }
  if (!P.crop) return;
  const int c = __syncthreads_count(keep);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}

// block_offsets: exclusive scan of block_counts (int64)
__global__ void __launch_bounds__(kCropThreads)
tnt_compact_kernel(const float* __restrict__ pts, const unsigned char* __restrict__ mask, int n,
                   const int64_t* __restrict__ block_offsets, float* __restrict__ out,
                   int64_t* __restrict__ out_index) {
  __shared__ int warp_base[kCropThreads / 32];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool keep = i < n && __ldg(mask + i);
  const unsigned b = __ballot_sync(0xffffffffu, keep);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_base[warp] = __popc(b);
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int w = 0; w < kCropThreads / 32; ++w) {
      const int c = warp_base[w];
      warp_base[w] = acc;
      acc += c;
    }
  }
  __syncthreads();
  if (!keep) return;
  const int64_t o = __ldg(block_offsets + blockIdx.x) + warp_base[warp] + __popc(b & ((1u << lane) - 1u));
  out[3 * o] = __ldg(pts + 3 * (size_t)i);
  out[3 * o + 1] = __ldg(pts + 3 * (size_t)i + 1);
  out[3 * o + 2] = __ldg(pts + 3 * (size_t)i + 2);
  if (out_index) out_index[o] = i;
}

// ---------------------------------------------------------------------------------- voxel mean
__global__ void __launch_bounds__(256)
tnt_voxel_mean_kernel(const float* __restrict__ pts, const int64_t* __restrict__ order,
                      const int* __restrict__ start, int nvox, float* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvox) return;
  const int b = __ldg(start + v), e = __ldg(start + v + 1);
  double s[3] = {0.0, 0.0, 0.0};
  for (int k = b; k < e; ++k) {
    const size_t p = (size_t)__ldg(order + k);
#pragma unroll
    for (int a = 0; a < 3; ++a) s[a] = __dadd_rn(s[a], (double)__ldg(pts + 3 * p + a));
  }
  const double cnt = (double)(e - b);
#pragma unroll
  for (int a = 0; a < 3; ++a) out[3 * (size_t)v + a] = __double2float_rn(__ddiv_rn(s[a], cnt));
}

// ---------------------------------------------------------------------------------- ICP moments
// sums: [count, sum d^2, sum s' (3), sum t' (3), sum |s'|^2, sum t'_a s'_b (9, row-major a)] with
// s' = s - origin, t' = t - origin over the sources i with index[i] >= 0, t = tgt[index[i]].
__global__ void __launch_bounds__(kMomThreads)
tnt_icp_moments_kernel(const float* __restrict__ src, int n, const float* __restrict__ tgt,
                       const int64_t* __restrict__ index, double ox, double oy, double oz,
                       double* __restrict__ partial) {
  double acc[kMoments];
#pragma unroll
  for (int k = 0; k < kMoments; ++k) acc[k] = 0.0;
  const double o[3] = {ox, oy, oz};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int64_t j = __ldg(index + i);
    if (j < 0) continue;
    double s[3], t[3], d[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double sa = (double)__ldg(src + 3 * (size_t)i + a);
      const double ta = (double)__ldg(tgt + 3 * (size_t)j + a);
      d[a] = __dsub_rn(ta, sa);
      s[a] = __dsub_rn(sa, o[a]);
      t[a] = __dsub_rn(ta, o[a]);
    }
    acc[0] = __dadd_rn(acc[0], 1.0);
    acc[1] = __dadd_rn(acc[1], __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])),
                                         __dmul_rn(d[2], d[2])));
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      acc[2 + a] = __dadd_rn(acc[2 + a], s[a]);
      acc[5 + a] = __dadd_rn(acc[5 + a], t[a]);
    }
    acc[8] = __dadd_rn(acc[8], __dadd_rn(__dadd_rn(__dmul_rn(s[0], s[0]), __dmul_rn(s[1], s[1])),
                                         __dmul_rn(s[2], s[2])));
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) acc[9 + 3 * a + b] = __dadd_rn(acc[9 + 3 * a + b], __dmul_rn(t[a], s[b]));
  }
  __shared__ double red[kMoments][kMomThreads];
#pragma unroll
  for (int k = 0; k < kMoments; ++k) red[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int w = kMomThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int k = 0; k < kMoments; ++k)
        red[k][threadIdx.x] = __dadd_rn(red[k][threadIdx.x], red[k][threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x < kMoments) partial[(size_t)blockIdx.x * kMoments + threadIdx.x] = red[threadIdx.x][0];
}

__global__ void __launch_bounds__(32)
tnt_icp_moments_final_kernel(const double* __restrict__ partial, int nblocks, double* __restrict__ out) {
  const int k = threadIdx.x;
  if (k >= kMoments) return;
  double s = 0.0;
  for (int b = 0; b < nblocks; ++b) s = __dadd_rn(s, partial[(size_t)b * kMoments + k]);
  out[k] = s;
}

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_tnt_crop_blocks(int n) { return n > 0 ? (n + kCropThreads - 1) / kCropThreads : 0; }

extern "C" int casmvs_tnt_transform_crop(const float* points, int n, const double* T,
                                         int axis, double axis_min, double axis_max,
                                         const double* polygon, int n_polygon, float* out,
                                         unsigned char* mask, int* block_counts, void* stream) {
  CASMVS_REQUIRE(n >= 0, "tnt_transform_crop: n < 0");
  CASMVS_REQUIRE(n == 0 || (points && out), "tnt_transform_crop: null pointer");
  CASMVS_REQUIRE(axis >= -1 && axis <= 2, "tnt_transform_crop: axis must be -1 (no crop), 0, 1 or 2");
  CropParams P;
  P.transform = T != nullptr;
  for (int k = 0; k < 12; ++k) P.T[k] = T ? T[k] : 0.0;
  P.crop = axis >= 0;
  P.axis = axis < 0 ? 0 : axis;
  P.amin = axis_min;
  P.amax = axis_max;
  P.m = n_polygon;
  if (P.crop) {
    CASMVS_REQUIRE(n_polygon >= 1 && n_polygon < (1 << 20), "tnt_transform_crop: bad polygon size");
    CASMVS_REQUIRE(n == 0 || (polygon && mask && block_counts), "tnt_transform_crop: null crop pointer");
  }
  if (n == 0) return 0;
  tnt_transform_crop_kernel<<<casmvs_tnt_crop_blocks(n), kCropThreads, 0, as_stream(stream)>>>(
      points, n, P, polygon, out, mask, block_counts);
  return after_launch("tnt_transform_crop");
}

extern "C" int casmvs_tnt_compact(const float* points, const unsigned char* mask, int n,
                                  const int64_t* block_offsets, float* out, int64_t* out_index,
                                  void* stream) {
  CASMVS_REQUIRE(n >= 0, "tnt_compact: n < 0");
  CASMVS_REQUIRE(n == 0 || (points && mask && block_offsets && out), "tnt_compact: null pointer");
  if (n == 0) return 0;
  tnt_compact_kernel<<<casmvs_tnt_crop_blocks(n), kCropThreads, 0, as_stream(stream)>>>(
      points, mask, n, block_offsets, out, out_index);
  return after_launch("tnt_compact");
}

extern "C" int casmvs_tnt_voxel_mean(const float* points, const int64_t* order,
                                     const int* voxel_start, int n_voxels, float* out,
                                     void* stream) {
  CASMVS_REQUIRE(n_voxels >= 0, "tnt_voxel_mean: n_voxels < 0");
  CASMVS_REQUIRE(n_voxels == 0 || (points && order && voxel_start && out),
                 "tnt_voxel_mean: null pointer");
  if (n_voxels == 0) return 0;
  tnt_voxel_mean_kernel<<<(n_voxels + 255) / 256, 256, 0, as_stream(stream)>>>(points, order,
                                                                             voxel_start, n_voxels, out);
  return after_launch("tnt_voxel_mean");
}

extern "C" size_t casmvs_tnt_icp_workspace_bytes(int n) {
  if (n < 0) return 0;
  const int nb = std::min(kMomMaxBlocks, std::max(1, (n + kMomThreads - 1) / kMomThreads));
  return (size_t)nb * kMoments * sizeof(double);
}

extern "C" int casmvs_tnt_icp_moments(const float* src, int n, const float* tgt, const int64_t* index,
                                      const double* origin3, double* moments, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  CASMVS_REQUIRE(n >= 0, "tnt_icp_moments: n < 0");
  CASMVS_REQUIRE(origin3, "tnt_icp_moments: null host array");
  CASMVS_REQUIRE(moments && workspace, "tnt_icp_moments: null pointer");
  CASMVS_REQUIRE(n == 0 || (src && tgt && index), "tnt_icp_moments: null pointer");
  CASMVS_REQUIRE(workspace_bytes >= casmvs_tnt_icp_workspace_bytes(n),
                 "tnt_icp_moments: workspace too small (%zu < %zu bytes)", workspace_bytes,
                 casmvs_tnt_icp_workspace_bytes(n));
  CASMVS_REQUIRE_ALIGNED("tnt_icp_moments: workspace", workspace, 8);
  cudaStream_t st = as_stream(stream);
  const int nb = (int)(casmvs_tnt_icp_workspace_bytes(n) / (kMoments * sizeof(double)));
  double* partial = static_cast<double*>(workspace);
  tnt_icp_moments_kernel<<<nb, kMomThreads, 0, st>>>(src, n, tgt, index, origin3[0], origin3[1],
                                                     origin3[2], partial);
  if (int rc = after_launch("tnt_icp_moments")) return rc;
  tnt_icp_moments_final_kernel<<<1, 32, 0, st>>>(partial, nb, moments);
  return after_launch("tnt_icp_moments_final");
}
