// View selection of a sparse reconstruction (MVSNet, Yao et al. 2018, §4.1): for every pair of
// images (i, j) the sum over the sparse points both see of a piecewise-Gaussian weight of the
// triangulation angle at the point,
//
//   s(i,j) = sum_{p : i,j in track(p)} G(theta_ij(p)),
//   theta_ij(p) = degrees(acos(clamp(dot(unit(c_i - p), unit(c_j - p)), -1, 1))),
//   G(theta) = exp(-(theta - 5)^2 / (2 * 1^2)) for theta <= 5, exp(-(theta - 5)^2 / (2 * 10^2)) else.
//
// All in double.  Deterministic: every s(i,j) is added in ascending point order.
//   1. a per-point pair count t(t-1)/2 and its exclusive scan give each point's first pair index
//      in the global pair enumeration (points ascending, then (a, b) with a < b row-major);
//   2. pair indices are processed in chunks of at most `chunk` entries: each entry finds its
//      point by binary search, computes its term and its key min(i,j) * n_img + max(i,j);
//   3. a stable radix sort by key keeps the entries of one key in pair-index order;
//   4. the first thread of each run loads the running sum of its key, adds the run's terms one by
//      one and stores it (both mirror elements).  Chunks run in pair-index order, so a chunked
//      call adds exactly the same terms in exactly the same order as a one-chunk call.
// The host reads the total pair count once (one stream synchronisation) to size the chunks.
#include <climits>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace casmvs {
namespace {

constexpr long long kDefaultChunk = 1ll << 22;   // pair entries per chunk (24 B each)
constexpr long long kMinChunk = 1ll << 10;

__global__ void pair_count_kernel(const long long* __restrict__ track_ptr, int n_pts,
                                  long long* __restrict__ count) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > n_pts) return;
  long long t = 0;
  if (p < n_pts) t = track_ptr[p + 1] - track_ptr[p];
  count[p] = t > 1 ? t * (t - 1) / 2 : 0;     // count[n_pts] = 0: the scan's last slot is the total
}

__device__ __forceinline__ double view_weight(double theta) {
  const double d = theta - 5.0;
  return theta <= 5.0 ? exp(-d * d / 2.0) : exp(-d * d / 200.0);
}

// one thread per pair entry g in [g0, g0 + n): its point, its two images and its term
__global__ void pair_expand_kernel(const double* __restrict__ centres, const double* __restrict__ points,
                                   const long long* __restrict__ track_ptr,
                                   const int* __restrict__ track_img,
                                   const long long* __restrict__ first, int n_img, int n_pts,
                                   long long g0, long long n, unsigned* __restrict__ keys,
                                   double* __restrict__ vals) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const long long g = g0 + e;
  // last point whose first pair index is <= g (points with no pairs share their successor's index)
  int lo = 0, hi = n_pts - 1;
  while (lo < hi) {
    const int mid = lo + (hi - lo + 1) / 2;
    if (first[mid] <= g) lo = mid; else hi = mid - 1;
  }
  const int p = lo;
  const long long base = track_ptr[p];
  const long long t = track_ptr[p + 1] - base;
  long long k = g - first[p];
  long long a = 0;
  while (k >= t - 1 - a) { k -= t - 1 - a; ++a; }
  const long long b = a + 1 + k;
  const int i = track_img[base + a], j = track_img[base + b];
  const unsigned sentinel = (unsigned)n_img * (unsigned)n_img;
  if (i < 0 || i >= n_img || j < 0 || j >= n_img || i == j) {
    keys[e] = sentinel;
    vals[e] = 0.0;
    return;
  }
  const double px = points[3 * p], py = points[3 * p + 1], pz = points[3 * p + 2];
  const double ax = centres[3 * i] - px, ay = centres[3 * i + 1] - py, az = centres[3 * i + 2] - pz;
  const double bx = centres[3 * j] - px, by = centres[3 * j + 1] - py, bz = centres[3 * j + 2] - pz;
  const double na = sqrt(ax * ax + ay * ay + az * az), nb = sqrt(bx * bx + by * by + bz * bz);
  double term = 0.0;                                   // a point on a camera centre has no angle
  if (na > 0.0 && nb > 0.0) {
    const double dot = (ax / na) * (bx / nb) + (ay / na) * (by / nb) + (az / na) * (bz / nb);
    const double theta = acos(fmin(fmax(dot, -1.0), 1.0)) * (180.0 / 3.14159265358979323846);
    term = view_weight(theta);
  }
  keys[e] = (unsigned)min(i, j) * (unsigned)n_img + (unsigned)max(i, j);
  vals[e] = term;
}

__global__ void run_sum_kernel(const unsigned* __restrict__ keys, const double* __restrict__ vals,
                               long long n, int n_img, double* __restrict__ scores) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const unsigned k = keys[e];
  const unsigned sentinel = (unsigned)n_img * (unsigned)n_img;
  if (k >= sentinel || (e > 0 && keys[e - 1] == k)) return;
  const unsigned i = k / (unsigned)n_img, j = k % (unsigned)n_img;
  double acc = scores[(size_t)i * n_img + j];
  for (long long r = e; r < n && keys[r] == k; ++r) acc += vals[r];
  scores[(size_t)i * n_img + j] = acc;
  scores[(size_t)j * n_img + i] = acc;
}

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

int key_end_bit(int n_img) {
  const unsigned long long top = (unsigned long long)n_img * n_img;   // sentinel, the largest key
  int bits = 1;
  while (bits < 32 && (top >> bits) != 0) ++bits;
  return bits;
}

// Workspace, each part 256-byte aligned: pair counts / first pair index (n_pts + 1 int64),
// keys, sorted keys (chunk uint32 each), values, sorted values (chunk doubles each), then the
// scan's or the sort's temporary storage, whichever is larger.
struct Layout {
  size_t off[6], total;     // off[5]: the temporary storage
};

bool layout(int n_img, int n_pts, long long chunk, Layout* L) {
  size_t scan_tmp = 0, sort_tmp = 0;
  if (cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (long long*)nullptr, (long long*)nullptr,
                                    n_pts + 1) != cudaSuccess)
    return false;
  if (cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const unsigned*)nullptr, (unsigned*)nullptr,
                                      (const double*)nullptr, (double*)nullptr, (int)chunk, 0,
                                      key_end_bit(n_img)) != cudaSuccess)
    return false;
  const size_t sizes[5] = {(size_t)(n_pts + 1) * 8, (size_t)chunk * 4, (size_t)chunk * 4,
                           (size_t)chunk * 8, (size_t)chunk * 8};
  L->off[0] = 0;
  for (int i = 0; i < 5; ++i) L->off[i + 1] = L->off[i] + align256(sizes[i]);
  L->total = L->off[5] + align256(scan_tmp > sort_tmp ? scan_tmp : sort_tmp);
  return true;
}

size_t bytes_for(int n_img, int n_pts, long long chunk) {
  Layout L;
  return layout(n_img, n_pts, chunk, &L) ? L.total : 0;
}

bool dims_ok(int n_img, int n_pts) {
  return n_img >= 0 && n_img <= 65535 && n_pts >= 0 && n_pts < INT_MAX;
}

}  // namespace
}  // namespace casmvs

using namespace casmvs;

extern "C" size_t casmvs_view_scores_workspace_bytes(int n_img, int n_pts, long long max_chunk_pairs) {
  if (!dims_ok(n_img, n_pts) || n_img < 2 || n_pts == 0) return 0;
  long long chunk = max_chunk_pairs > 0 ? max_chunk_pairs : kDefaultChunk;
  if (chunk < kMinChunk) chunk = kMinChunk;
  if (chunk > kDefaultChunk) chunk = kDefaultChunk;
  return bytes_for(n_img, n_pts, chunk);
}

extern "C" int casmvs_view_scores_fwd(const double* centres, const double* points,
                                      const long long* track_ptr, const int* track_img, int n_img,
                                      int n_pts, double* scores, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  CASMVS_REQUIRE(dims_ok(n_img, n_pts), "view_scores: bad dims (n_img %d, n_pts %d)", n_img, n_pts);
  if (n_img == 0) return 0;
  CASMVS_REQUIRE(scores, "view_scores: null pointer (scores)");
  cudaStream_t st = as_stream(stream);
  const size_t out_bytes = (size_t)n_img * n_img * sizeof(double);
  if (n_img < 2 || n_pts == 0) {
    if (cudaMemsetAsync(scores, 0, out_bytes, st) != cudaSuccess)
      return after_launch("view_scores memset");
    return 0;
  }
  CASMVS_REQUIRE(centres && points && track_ptr && track_img && workspace,
                 "view_scores: null pointer");
  CASMVS_REQUIRE_ALIGNED("view_scores", workspace, 256);
  CASMVS_REQUIRE_ALIGNED("view_scores", centres, 8);
  CASMVS_REQUIRE_ALIGNED("view_scores", points, 8);
  CASMVS_REQUIRE_ALIGNED("view_scores", track_ptr, 8);
  CASMVS_REQUIRE_ALIGNED("view_scores", track_img, 4);
  CASMVS_REQUIRE_ALIGNED("view_scores", scores, 8);
  // the largest chunk (power-of-two steps down from the default) the workspace holds
  long long chunk = kDefaultChunk;
  while (chunk > kMinChunk && bytes_for(n_img, n_pts, chunk) > workspace_bytes) chunk /= 2;
  const size_t need = bytes_for(n_img, n_pts, chunk);
  CASMVS_REQUIRE(need && workspace_bytes >= need,
                 "view_scores: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
  Layout L;
  layout(n_img, n_pts, chunk, &L);
  char* ws = static_cast<char*>(workspace);
  long long* first = reinterpret_cast<long long*>(ws + L.off[0]);
  unsigned* keys = reinterpret_cast<unsigned*>(ws + L.off[1]);
  unsigned* keys_sorted = reinterpret_cast<unsigned*>(ws + L.off[2]);
  double* vals = reinterpret_cast<double*>(ws + L.off[3]);
  double* vals_sorted = reinterpret_cast<double*>(ws + L.off[4]);
  void* tmp = ws + L.off[5];
  const size_t tmp_bytes = workspace_bytes - L.off[5];

  if (cudaMemsetAsync(scores, 0, out_bytes, st) != cudaSuccess)
    return after_launch("view_scores memset");
  pair_count_kernel<<<(unsigned)((n_pts + 1 + 255) / 256), 256, 0, st>>>(track_ptr, n_pts, first);
  if (int rc = after_launch("view_scores count")) return rc;
  size_t scan_bytes = tmp_bytes;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, first, first, n_pts + 1, st);
  if (e != cudaSuccess) {
    set_error("view_scores: scan failed: %s", cudaGetErrorString(e));
    return -2;
  }
  if (int rc = after_launch("view_scores scan")) return rc;
  long long total = 0;
  e = cudaMemcpyAsync(&total, first + n_pts, sizeof(total), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    set_error("view_scores: reading the pair count failed: %s", cudaGetErrorString(e));
    return -2;
  }
  const int end_bit = key_end_bit(n_img);
  for (long long g0 = 0; g0 < total; g0 += chunk) {
    const long long n = total - g0 < chunk ? total - g0 : chunk;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    pair_expand_kernel<<<blocks, 256, 0, st>>>(centres, points, track_ptr, track_img, first, n_img,
                                               n_pts, g0, n, keys, vals);
    if (int rc = after_launch("view_scores expand")) return rc;
    size_t sort_bytes = tmp_bytes;
    e = cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, keys, keys_sorted, vals, vals_sorted,
                                        (int)n, 0, end_bit, st);
    if (e != cudaSuccess) {
      set_error("view_scores: radix sort failed: %s", cudaGetErrorString(e));
      return -2;
    }
    if (int rc = after_launch("view_scores sort")) return rc;
    run_sum_kernel<<<blocks, 256, 0, st>>>(keys_sorted, vals_sorted, n, n_img, scores);
    if (int rc = after_launch("view_scores sum")) return rc;
  }
  return 0;
}
