// TMA helpers shared by the TMA-fed tensor-core convolution kernels (sm_90a).
#pragma once
#include <cuda.h>
#include <stdlib.h>

#include "tc_common.cuh"

namespace casmvs {
namespace tma {

__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "r"(c4)
      : "memory");
}

// Weight image -> shared memory as 1-D bulk copies issued by ONE thread and completed on an
// mbarrier (armed here with the byte count): the CTA's other warps go straight to their roles
// and only the MMA issuer waits for it, so the (14-110 KB) image fetch overlaps the first
// input-brick loads instead of preceding them.  bytes % 16 == 0, both sides 16 B aligned.
__device__ __forceinline__ void load_image_bulk(uint32_t dst_smem, const float* src, int bytes,
                                                uint32_t bar) {
  mbar_expect_tx(bar, (uint32_t)bytes);
  for (int off = 0; off < bytes; off += 32768) {
    const uint32_t n = (uint32_t)(bytes - off < 32768 ? bytes - off : 32768);
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(dst_smem + off), "l"(reinterpret_cast<const char*>(src) + off), "r"(n), "r"(bar)
        : "memory");
  }
}

// Programmatic dependent launch: the kernels are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, so a CTA may start while the previous
// kernel of the stream is still draining.  Everything before pdl_wait() -- barrier init,
// the weight-image bulk copy, parameter loads: nothing that depends on the previous
// kernel's output -- overlaps that tail; pdl_wait() returns once the previous grid has completed
// and its writes are visible.  pdl_trigger() lets the next kernel of the stream do the same.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
// Launch helper: <<<>>> semantics plus the programmatic-serialization attribute (CASMVS_PDL=0:
// plain stream order, in which case the two instructions above are no-ops).  allow = false on
// the call that has just launched the weight-image builder: the prologue reads that image.
template <typename Kernel, typename... Args>
inline cudaError_t launch_pdl(bool allow, Kernel kfn, dim3 grid, int threads, size_t smem,
                              cudaStream_t st, Args... args) {
  static int pdl = -1;
  if (pdl < 0) {
    const char* e = getenv("CASMVS_PDL");
    pdl = e ? atoi(e) : 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (pdl && allow) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kfn, args...);
}

// Tiled tensor map over the activation tensor x (B,D,H,W,C) viewed as {C, W, H, D, B} with box
// {CB, box_w, box_h, 1, 1}, swizzle = CB*4 bytes (128/64/32; none for the 16-byte boxes of the
// conv kernels), out-of-bounds elements zero-filled
// (= the convolution's zero padding).  stride_w = 2: the box walks every second voxel along W
// (box_w counts traversed positions, so ceil(box_w / 2) voxels are loaded): the even / odd
// column planes of the stride-2 convolutions.  Memoised by (pointer, shape, box); null +
// casmvs error when the driver entry point is missing or the encode fails.  (conv3d_tma.cu)
//
// blocked = true: x is stored blocked by channel quads, (B, C/4, D, H, W, 4) fp32 (CB must be
// 4), so a row of box_w voxels of one quad is 16 box_w contiguous bytes.  The map writes the
// same [box_h][box_w][4] brick to shared memory as the channels-last one; only the load
// coordinates differ (brick_coords).
const CUtensorMap* input_map(const float* x, int B, int D, int H, int W, int C, int CB, int box_w,
                             int box_h, int stride_w = 1, bool blocked = false);

// Load coordinates of the brick of channel quad q whose first voxel is (w, h, d) of batch item
// b, for the map input_map built (cq = C/4).  Blocked, stride 1: {4w, h, d, q, b}; blocked,
// stride 2: {0, w, h, d, b cq + q}; channels-last: {4q, w, h, d, b}.
struct Coords5 { int c[5]; };
__host__ __device__ __forceinline__ Coords5 brick_coords(bool blocked, int stride_w, int cq, int q,
                                                         int w, int h, int d, int b) {
  if (!blocked) return {{4 * q, w, h, d, b}};
  if (stride_w == 1) return {{4 * w, h, d, q, b}};
  return {{0, w, h, d, b * cq + q}};
}

// Element offset of channel c of voxel (b, d, h, w) in a (B, D, H, W, C) volume stored
// channels-last or blocked by channel quads (C % 4 == 0 when blocked).  Channels c and c + 1
// with c even are adjacent in both layouts.
__host__ __device__ __forceinline__ size_t vol_offset(bool blocked, int b, int d, int h, int w,
                                                      int c, int D, int H, int W, int C) {
  if (!blocked) return ((((size_t)b * D + d) * H + h) * W + w) * C + c;
  return (((((size_t)b * (C >> 2) + (c >> 2)) * D + d) * H + h) * W + w) * 4 + (c & 3);
}

// Generic fp32 tiled map (rank <= 5, unit element strides, zero fill out of bounds); dims /
// box innermost first, strides_bytes for dims 1..rank-1.  0 on success.  (conv3d_tma.cu)
int encode_tiled(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}

inline int pow2_floor(int v) { int r = 1; while (r * 2 <= v) r *= 2; return r; }

// Resident CTAs per SM of a persistent kernel (registers and shared memory), at least 1.
template <typename K>
inline int resident_per_sm(K kfn, int threads, int smem) {
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kfn, threads, smem) != cudaSuccess) n = 1;
  return n < 1 ? 1 : n;
}

// Depth-chunk length for the persistent kernels.  An item (tile column x depth chunk of dc
// output groups) costs mul*dc + add input slices (+ `fixed` for pipeline fill / drain); CTA k
// runs items k, k + resident, ...: the kernel lasts as long as the busiest CTA, i.e.
// ceil(items / resident) items.  Long chunks amortise the depth halo, short ones fill the
// machine and balance the last round; pick the cheapest (ties -> longer chunks).
inline int pick_dchunk(int D, int cap, long cols, long resident, int mul, int add, int fixed = -1) {
  if (fixed < 0) {                      // CASMVS_DCHUNK_FIXED: per-item overhead in slice units
    static int env_fixed = -1;
    if (env_fixed < 0) {
      const char* e = getenv("CASMVS_DCHUNK_FIXED");
      env_fixed = e ? atoi(e) : 0;   // measured on cfg2: 0 -> 1.0876, 1 -> 1.0888, 2 -> 1.0938 ms/step
    }
    fixed = env_fixed;
  }
  if (cap > D) cap = D;
  if (cap < 1) cap = 1;
  if (resident < 1) resident = 1;
  int best = cap;
  long best_cost = -1;
  for (int dc = cap; dc >= 1; --dc) {
    const long items = cols * ((D + dc - 1) / dc);
    const long rounds = (items + resident - 1) / resident;
    const long cost = rounds * (mul * dc + add + fixed);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = dc; }
  }
  return best;
}

}  // namespace tma
}  // namespace casmvs
