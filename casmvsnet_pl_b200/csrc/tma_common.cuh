// TMA helpers shared by the TMA-fed tensor-core convolution kernels (sm_90a).
#pragma once
#include <cuda.h>

#include "tc_common.cuh"

namespace casmvs {
namespace tma {

using namespace tc;

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
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (switches().pdl && allow) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kfn, args...);
}

// A tiled tensor map of fp32 elements, out-of-bounds elements zero-filled: dims, box and element
// strides innermost first, byte strides for dims 1 .. rank-1, swizzle in bytes (0: none).
// Value-initialise it (`MapDesc d{};`): unused entries must be zero, since maps are memoised by
// the whole description.
struct MapDesc {
  const void* base;
  int rank, swizzle_bytes;
  uint64_t dims[5], strides_bytes[4];
  uint32_t box[5], elem_strides[5];
};
// Encodes d into *out.  Tensor maps are pure functions of their description, and inference
// encodes the same ones every step (same workspace pointers), so they are memoised.  0, or -2
// with the casmvs error set.  (conv3d_tma.cu)
int encode_map(const MapDesc& d, CUtensorMap* out);

// The map of a conv kernel's input x (B,D,H,W,C): a box of one channel quad, box_w x box_h
// voxels of one slice (16 bytes per voxel, no swizzle).  Two forms:
//   * channels-last: {C, W, H, D, B}, box {4, box_w, box_h, 1, 1};
//   * blocked by channel quads, (B, C/4, D, H, W, 4) fp32: {4W, H, D, C/4, B}, box
//     {4 box_w, box_h, 1, 1, 1} -- the quad folded into the inner dimension, so one brick row
//     is 16 box_w contiguous bytes.
// stride_w = 2 (channels-last only): the box walks every second voxel along W (box_w counts
// traversed positions, so ceil(box_w / 2) voxels are loaded): the even / odd column planes of
// the stride-2 convolutions.  Both forms write the same [box_h][box_w][4] brick to shared
// memory; only the load coordinates differ (brick_coords).  0, or -2 with the casmvs error set.
// (conv3d_tma.cu)
int input_map(CUtensorMap* out, const float* x, int B, int D, int H, int W, int C, int box_w,
              int box_h, int stride_w = 1, bool blocked = false);

// Load coordinates of the brick of channel quad q whose first voxel is (w, h, d) of batch item
// b, for the map input_map built.  Blocked: {4w, h, d, q, b}; channels-last: {4q, w, h, d, b}.
struct Coords5 { int c[5]; };
__host__ __device__ __forceinline__ Coords5 brick_coords(bool blocked, int q, int w, int h, int d,
                                                         int b) {
  if (!blocked) return {{4 * q, w, h, d, b}};
  return {{4 * w, h, d, q, b}};
}

// Element offset of channel c of voxel (b, d, h, w) in a (B, D, H, W, C) volume stored
// channels-last or blocked by channel quads (C % 4 == 0 when blocked).  Channels c and c + 1
// with c even are adjacent in both layouts.
__host__ __device__ __forceinline__ size_t vol_offset(bool blocked, int b, int d, int h, int w,
                                                      int c, int D, int H, int W, int C) {
  if (!blocked) return ((((size_t)b * D + d) * H + h) * W + w) * C + c;
  return (((((size_t)b * (C >> 2) + (c >> 2)) * D + d) * H + h) * W + w) * 4 + (c & 3);
}

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}

// ---- the pipeline of the persistent TMA conv kernels (conv3d_tma.cu, conv3d_tma2.cu,
// conv3d_tail.cu) ----

// A ring of SLOTS shared-memory slots, each guarded by a "full" and an "empty" mbarrier (arrays
// of 8-byte barriers).  Slices are numbered g = 0, 1, ... over the CTA's whole run, across work
// items, so slot g % SLOTS is in phase g / SLOTS: its producer waits for the consumers to have
// released phase g / SLOTS - 1, its consumers for phase g / SLOTS to be filled.
template <int SLOTS>
struct Ring {
  uint32_t full, empty;
  // barrier t < 2 SLOTS (full 0 .. SLOTS-1, then empty; t >= 2 SLOTS: none), so that threads
  // 0 .. 2 SLOTS-1 can initialise one each; fence_barrier_init() after it
  __device__ __forceinline__ void init(uint32_t t, uint32_t full_arrivals,
                                       uint32_t empty_arrivals) const {
    if (t < SLOTS) mbar_init(full + 8 * t, full_arrivals);
    else if (t < 2 * SLOTS) mbar_init(empty + 8 * (t - SLOTS), empty_arrivals);
  }
  __device__ __forceinline__ uint32_t full_bar(uint32_t g) const { return full + 8 * (g % SLOTS); }
  // producer: wait until slot g is free, return it (a TMA producer then arms full_bar(g) with
  // expect_tx; a generic-proxy one writes the slot and calls publish)
  __device__ __forceinline__ int acquire(uint32_t g) const {
    const int slot = g % SLOTS;
    if (g >= (uint32_t)SLOTS) mbar_wait(empty + 8 * slot, ((g / SLOTS) - 1) & 1);
    return slot;
  }
  __device__ __forceinline__ void publish(uint32_t g) const { mbar_arrive(full_bar(g)); }
  // consumer: wait until slot g is filled, return it; release it once this thread's reads are done
  __device__ __forceinline__ int wait(uint32_t g) const {
    mbar_wait(full_bar(g), (g / SLOTS) & 1);
    return g % SLOTS;
  }
  __device__ __forceinline__ void release(uint32_t g) const { mbar_arrive(empty + 8 * (g % SLOTS)); }
};

// The dynamic shared memory rounded up to 1024 B (every layout reserves 1024 B of slack): its
// shared-space address, and its generic pointer in *smem.
__device__ __forceinline__ uint32_t smem_align_1024(unsigned char* raw, unsigned char** smem) {
  const uint32_t r = smem_u32(raw);
  const uint32_t base = (r + 1023u) & ~1023u;
  *smem = raw + (base - r);
  return base;
}

// Per-channel scale [N] and shift [N] of this CTA's output channels co_base .. co_base + cout - 1
// (null scale: 1, null shift: 0), zero beyond cout.
template <int N>
__device__ __forceinline__ void stage_scale_shift(float* s, const float* scale, const float* shift,
                                                  int co_base, int cout) {
  for (int i = threadIdx.x; i < N; i += kConvThreads) {
    s[i] = (i < cout) ? (scale ? __ldg(scale + co_base + i) : 1.f) : 0.f;
    s[N + i] = (i < cout) ? (shift ? __ldg(shift + co_base + i) : 0.f) : 0.f;
  }
}

// A weight image to bring to shared memory: load_image_bulk's arguments.
struct ImageCopy { uint32_t dst; const float* src; int bytes; uint32_t bar; };

// The end of the CTA prologue.  The barrier inits and shared-memory writes above become visible
// to the async proxy and to every thread, thread 0 starts the weight-image copies, and the CTA
// lets the next kernel of the stream start and then waits for the previous one: nothing before
// this call may read the previous kernel's output.
template <typename... Images>
__device__ __forceinline__ void end_prologue(const Images&... img) {
  fence_proxy_async();
  __syncthreads();
  if (threadIdx.x == 0) (load_image_bulk(img.dst, img.src, img.bytes, img.bar), ...);
  pdl_trigger();
  pdl_wait();
}

// The work of a persistent kernel: for each batch item, depth chunks of dchunk M-space slices
// times tiles of kTileH x kTileW voxels.  The CTA of blockIdx.x runs items blockIdx.x,
// blockIdx.x + gridDim.x, ...
struct Work { int tiles_w, tiles_h, nchunks, dchunk; };
struct Item { int b, chunk, h0, w0; };
__device__ __forceinline__ Item decode_item(int item, const Work& w) {
  const int tw = item % w.tiles_w; item /= w.tiles_w;
  const int th = item % w.tiles_h; item /= w.tiles_h;
  return {item / w.nchunks, item % w.nchunks, th * kTileH, tw * kTileW};
}

// Resident CTAs per SM of a persistent kernel (registers and shared memory), at least 1.
template <typename K>
inline int resident_per_sm(K kfn, int threads, int smem) {
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kfn, threads, smem) != cudaSuccess) n = 1;
  return n < 1 ? 1 : n;
}

// Depth-chunk length for the persistent kernels.  An item (tile column x depth chunk of dc
// output groups) costs mul*dc + add input slices; CTA k runs items k, k + resident, ...: the
// kernel lasts as long as the busiest CTA, i.e. ceil(items / resident) items.  Long chunks
// amortise the depth halo, short ones fill the machine and balance the last round; pick the
// cheapest (ties -> longer chunks).  Charging a further 1 or 2 slices per item for pipeline fill
// was measured slower on cfg2 (1.0876 -> 1.0888 / 1.0938 ms per step).
inline int pick_dchunk(int D, int cap, long cols, long resident, int mul, int add) {
  if (cap > D) cap = D;
  if (cap < 1) cap = 1;
  if (resident < 1) resident = 1;
  int best = cap;
  long best_cost = -1;
  for (int dc = cap; dc >= 1; --dc) {
    const long items = cols * ((D + dc - 1) / dc);
    const long rounds = (items + resident - 1) / resident;
    const long cost = rounds * (mul * dc + add);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = dc; }
  }
  return best;
}

// Launch size of a persistent kernel (kConvThreads threads, `smem` bytes of shared memory) whose
// nco Cout chunks run side by side (grid.y): `cols` tile columns (batch items x tiles) over an
// M-space depth `depth`, chunked by pick_dchunk(cap, mul, add) or, when 1 <= n <= cap, by
// CASMVS_TMA_DCHUNK=n; at most as many CTAs along x as are resident at once.
struct Sizing { int dchunk, nchunks; dim3 grid; };
template <typename K>
inline Sizing size_persistent(K kfn, int smem, int nco, long cols, int depth, int cap, int mul,
                              int add) {
  long resident = (long)num_sms() * resident_per_sm(kfn, kConvThreads, smem) / nco;
  int dc = pick_dchunk(depth, cap, cols, resident, mul, add);
  const int dc_env = switches().tma_dchunk;
  if (dc_env > 0 && dc_env <= cap) dc = dc_env < depth ? dc_env : depth;
  if (resident < 1) resident = 1;
  const int nchunks = (depth + dc - 1) / dc;
  const long items = cols * nchunks;
  return {dc, nchunks, dim3((unsigned)(items < resident ? items : resident), (unsigned)nco)};
}

}  // namespace tma
}  // namespace casmvs
