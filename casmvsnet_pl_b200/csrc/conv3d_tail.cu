// K2 tail — CostRegNet's conv11 (transposed 16 -> 8, + the c0 skip) and prob head (8 -> 1) as
// one kernel: the logits are computed from u9 and c0, and the full-resolution u11 volume lives
// only in shared memory.  sm_90a, wgmma tf32, fp32 accumulators in registers.
//
// Replaces (reference): conv0 + conv11(x) and prob(x), models/mvsnet.py:101,103.
//
// Bit-identical to conv3d_tma2_kernel<MODE_T, 16, 8> followed by conv3d_tma_kernel<8, 8, *,
// false>: every u11 value is made by the same wgmma (m64n96k8, same B image, same tap / k8
// order, same accumulator roll) and the same epilogue (scale/shift, LeakyReLU, + c0, tf32
// rounding).  Every logit is the same sum: prob's image has Cout = 1 in each GW = 8 column
// group, so of its m64n24k8 only columns 0, 8 and 16 (kd = 2, 1, 0) are live.  Here those three
// columns sit side by side in one m64n8k8, with the same A operand, the same tap / k8 order and
// the same rolling window, a third of the tensor work.
//
// Work item: a prob output tile of 8(w) x 16(h) voxels (tc::kTileW x kTileH) times a chunk of
// output slices [d0, d1), d0 and d1 even.  Its prob GEMM reads u11 over the 18 x 10 halo region
// of slices d0-1 .. d1; those u11 voxels come from the u9 voxels of an 11 x 6 region (output
// 2j + p reads input j and j + 1), u9 slices d0/2-1 .. d1/2.
//   * Producer warp: per u9 slice ("step") one TMA load per u9 channel quad of the 11 x 6 brick
//     into the u9 ring, and the c0 skip bricks ([18][10][4], the stride-1 kernel's box) of the
//     two u11 slices the step completes into the c0 ring.  Out-of-range voxels are zero-filled
//     by the TMA unit.
//   * Warpgroup 0 (conv11): the u9 brick is stored row after row, 6 voxels each, so GEMM row m
//     is u9 voxel m of the flattened region and 8 consecutive rows are one 128-byte core matrix:
//     M = 64 covers the 60 voxels the region needs.  Tap (sh, sw) is the view shifted by
//     6 sh + sw voxels; rows whose shifted view wraps into the next brick row only feed u11
//     voxels outside the 18 x 10 region, which are never stored.  After step s the accumulator
//     holds u11 slices 2s-1 (classes pd = 1) and 2s (pd = 0): their epilogue writes the u11
//     bricks of a ring in shared memory, with u11 voxels outside the volume set to zero (prob's
//     zero padding).  The wgmma of u9 slice -1 are skipped: it only feeds u11 slices -3 .. -1.
//   * Warpgroup 1 (prob): per u11 slice, the stride-1 GEMM (N = 8: the three kd columns) for
//     both 64-row halves of the tile; the logits of the output slice the previous u11 slice completed are stored while
//     those wgmma execute (carried across items, as in conv3d_tma.cu).  The wgmma of u11 slice
//     -1 (all zero) are skipped: the only stored column it feeds holds +0 and stays so.
#include "common.cuh"
#include "tc_common.cuh"
#include "tma_common.cuh"

namespace casmvs {

// conv3d_tma.cu / conv3d_tma2.cu: the operand images of prob and conv11, shared through the
// image cache with the unfused layers
int conv3d_tma_prob_image(const float* wpk, cudaStream_t st, tc::ImageRef* ir);
int conv3d_tma2_conv11_image(const float* wpk, cudaStream_t st, tc::ImageRef* ir);

namespace tail {

using namespace tc;
using namespace tma;

struct Params {
  const float* img11;    // conv11 B image (conv3d_tma2 MODE_T, CIN 16, COUT 8)
  const float* imgp;     // prob B image (conv3d_tma stride-1, CIN 8, GW 8)
  const float *scale11, *shift11, *scalep, *shiftp;
  float* logits;         // (B,D,H,W)
  float slope;           // conv11's LeakyReLU slope
  int B, D, H, W;        // full resolution: c0, u11, logits
  Work work;             // prob output tiles; dchunk even
};

constexpr int kU9W = 6, kU9H = 11;                                  // u9 brick columns, rows
constexpr int kU9Data = kU9H * kU9W * 16;
constexpr int kU9Bytes = (kU9Data + 127) / 128 * 128;
constexpr int kBrickData = kHaloH * kHaloW * 16;                    // c0 / u11 brick, one quad
constexpr int kBrickBytes = (kBrickData + 127) / 128 * 128;
constexpr int kSliceBytes = 2 * kBrickBytes;                        // 8 channels of one slice
constexpr int kU9SlotBytes = 4 * kU9Bytes;                         // u9 slice, 16 channels
constexpr int kC0SlotBytes = 2 * kSliceBytes;                       // 2 c0 slices
// The u9 slot of a step is released once its wgmma retire, its c0 slot only after the epilogue
// has read the skip: separate rings, so the next u9 loads need not wait for the epilogue.
constexpr int U9_SLOTS = 4, C0_SLOTS = 3, U_SLOTS = 4;
constexpr int kW11Bytes = 4 * 16 * 96 * 4;                          // [tap][cq][12 COUT][4]
constexpr int kWpBytes = 9 * 8 * 24 * 4;                            // [kh][kw][cq][3 GW][4]
constexpr int kU9Off = 0;
constexpr int kC0Off = kU9Off + U9_SLOTS * kU9SlotBytes;
constexpr int kUOff = kC0Off + C0_SLOTS * kC0SlotBytes;
constexpr int kW11Off = kUOff + U_SLOTS * kSliceBytes;
constexpr int kWpOff = kW11Off + kW11Bytes;
// prob's three kd columns (column 0 of each GW = 8 group of the image above) side by side in
// one 8-column group: [kh][kw][cq][8][4], columns 3 .. 7 zero
constexpr int kWp8Bytes = 9 * 8 * 8 * 4;
constexpr int kWp8Off = kWpOff + kWpBytes;
constexpr int kParamOff = kWp8Off + kWp8Bytes;                      // scale11, shift11, prob
constexpr int kBarOff = kParamOff + 4 * 8 * 4;
// barriers: u9_full[4] @0, u9_empty[4] @32, c0_full[4] @64, c0_empty[4] @96, u_full[4] @128,
// u_empty[4] @160, w11 @192, wp @200
constexpr int kTotal = kBarOff + 256 + 1024;                        // + alignment slack
static_assert(U9_SLOTS <= 4 && C0_SLOTS <= 4 && U_SLOTS <= 4, "barrier slots");
static_assert(kU9SlotBytes % 128 == 0 && kSliceBytes % 128 == 0, "128-byte aligned slots");

// two CTAs per SM (registers <= 96, 2 x 110 KB of shared memory)
__device__ __forceinline__ float opaque_zero() {
  float z;
  asm volatile("mov.b32 %0, 0;" : "=f"(z));
  return z;
}

// The value of lane + 1.  The read of v is a volatile asm, so it stays after the preceding
// wgmma_wait_all: a plain shuffle's operand move is hoisted above the commit, and ptxas then
// waits for the slice's wgmma there (C7517), before the pending epilogue.
__device__ __forceinline__ float shfl_down_1(float v) {
  uint32_t b;
  asm volatile("mov.b32 %0, %1;" : "=r"(b) : "f"(v));
  return __uint_as_float(__shfl_down_sync(0xffffffffu, b, 1));
}

__global__ void __launch_bounds__(kConvThreads, 2)
conv3d_tail_kernel(const __grid_constant__ CUtensorMap u9map,
                   const __grid_constant__ CUtensorMap c0map, const Params p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem;
  const uint32_t s_base = smem_align_1024(smem_raw, &smem);
  const uint32_t s_u9 = s_base + kU9Off, s_c0 = s_base + kC0Off, s_u = s_base + kUOff,
                 s_w11 = s_base + kW11Off, s_wp = s_base + kWpOff, s_bar = s_base + kBarOff;
  float* s_param = reinterpret_cast<float*>(smem + kParamOff);
  // u9 and c0 input slots, filled by TMA; u11 slices, written by warpgroup 0 and read by
  // warpgroup 1
  const Ring<U9_SLOTS> u9_ring{s_bar, s_bar + 32};
  const Ring<C0_SLOTS> c0_ring{s_bar + 64, s_bar + 96};
  const Ring<U_SLOTS> u_ring{s_bar + 128, s_bar + 160};
  const uint32_t bar_w11 = s_bar + 192, bar_wp = s_bar + 200;
  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int total_items = p.B * p.work.nchunks * p.work.tiles_h * p.work.tiles_w;

  // ---- one-time setup ----
  if (threadIdx.x == 0) {                           // thread 0 initialises every barrier
    for (int t = 0; t < 2 * U9_SLOTS; ++t) u9_ring.init(t, 1, 128);
    for (int t = 0; t < 2 * C0_SLOTS; ++t) c0_ring.init(t, 1, 128);
    for (int t = 0; t < 2 * U_SLOTS; ++t) u_ring.init(t, 128, 128);
    mbar_init(bar_w11, 1);
    mbar_init(bar_wp, 1);
    fence_barrier_init();
  }
  if (threadIdx.x < 8) {
    const int i = threadIdx.x;
    s_param[i] = __ldg(p.scale11 + i);
    s_param[8 + i] = __ldg(p.shift11 + i);
    s_param[16 + i] = i < 1 ? __ldg(p.scalep) : 0.f;           // prob: Cout = 1 of GW = 8
    s_param[24 + i] = i < 1 ? __ldg(p.shiftp) : 0.f;
  }
  // The TMA loads never write the tail of a u9 brick (voxels 66 .. 71), but the shifted views of
  // GEMM rows 59 .. 63 read it, times the zero weight rows of the classes a tap does not reach:
  // it must hold finite values, or 0 x NaN would reach u11 voxels of the region.
  for (int i = threadIdx.x; i < U9_SLOTS * 4 * (kU9Bytes - kU9Data) / 16; i += kConvThreads) {
    const int per = (kU9Bytes - kU9Data) / 16, brick = i / per;
    *reinterpret_cast<float4*>(smem + kU9Off + brick * kU9Bytes + kU9Data + (i % per) * 16) =
        make_float4(0.f, 0.f, 0.f, 0.f);
  }
  end_prologue(ImageCopy{s_w11, p.img11, kW11Bytes, bar_w11},
               ImageCopy{s_wp, p.imgp, kWpBytes, bar_wp});
  bool w_ready = false;                             // consumers: weight image has landed
  const int wl = warp & 3;
  // An item: batch item b, prob tile (h0, w0), output slices d0 .. d0 + nd - 1 (nd even), read
  // from u9 slices s0 .. s0 + nsteps - 1 = d0/2 - 1 .. d1/2.  Each role walks the CTA's items
  // itself; its slice counts (and warpgroup 1's pending logits) run on across items.
  struct Chunk { int b, h0, w0, d0, nd, s0, nsteps; };
  auto chunk_of = [&](int item) {
    const Item t = decode_item(item, p.work);
    const int d0 = t.chunk * p.work.dchunk, nd = min(p.D, d0 + p.work.dchunk) - d0;
    return Chunk{t.b, t.h0, t.w0, d0, nd, d0 / 2 - 1, nd / 2 + 2};
  };

  if (warp == kProdWarp) {
    // ============ producer: 4 u9 loads per step, + 2 x 2 c0 loads after the first ============
    if (lane == 0) {
      uint32_t gin = 0, gc = 0;                     // steps / c0 slot fills before this item
      for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
        const Chunk t = chunk_of(item);
        for (int st = 0; st < t.nsteps; ++st) {
          const uint32_t g = gin + st;
          const uint32_t dst = s_u9 + u9_ring.acquire(g) * kU9SlotBytes, full = u9_ring.full_bar(g);
          mbar_expect_tx(full, 4 * kU9Data);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const Coords5 k = brick_coords(true, q, t.w0 / 2 - 1, t.h0 / 2 - 1, t.s0 + st, t.b);
            tma_load_5d(dst + q * kU9Bytes, &u9map, full, k.c[0], k.c[1], k.c[2], k.c[3], k.c[4]);
          }
          if (st > 0) {                             // the first step's u11 slices are not used
            const uint32_t gs = gc + st - 1;
            const uint32_t dc0 = s_c0 + c0_ring.acquire(gs) * kC0SlotBytes,
                           fc0 = c0_ring.full_bar(gs);
            mbar_expect_tx(fc0, 4 * kBrickData);
#pragma unroll
            for (int k2 = 0; k2 < 2; ++k2) {
#pragma unroll
              for (int q = 0; q < 2; ++q) {
                const Coords5 k = brick_coords(true, q, t.w0 - 1, t.h0 - 1,
                                               2 * (t.s0 + st) - 1 + k2, t.b);
                tma_load_5d(dc0 + k2 * kSliceBytes + q * kBrickBytes, &c0map, fc0, k.c[0], k.c[1],
                            k.c[2], k.c[3], k.c[4]);
              }
            }
          }
        }
        gin += t.nsteps;
        gc += t.nsteps - 1;
      }
    }
    __syncwarp();
  } else if (warp < 4) {
    // ===================== warpgroup 0: conv11 into the u11 ring =====================
    constexpr uint32_t a_lbo = kU9Bytes, a_sbo = 128;            // next quad; next 8 voxels
    constexpr uint32_t b_lbo = 96 * 16, b_sbo = 128;
    const uint64_t a_desc0 = make_desc(s_u9, a_lbo, a_sbo);
    const uint64_t b_desc0 = make_desc(s_w11, b_lbo, b_sbo);
    // [kd=0 block of group s-1 | kd=1 block of group s | kd=2 block of group s], as in
    // conv3d_tma2's MODE_T (each block: 4 classes x 8 channels)
    float acc[48];
#pragma unroll
    for (int i = 0; i < 48; ++i) acc[i] = 0.f;
    // This thread's 8 column pairs of a block (for_each_pair order: class j, row half h)
    // hold channels c, c + 1 of u9 voxel m = 16 wl + lane/4 + 8h, class (ph, pw) = j: output
    // voxel (2 jr + ph - 1, 2 jc + pw - 1) of the 18 x 10 region, jr, jc = m / 6, m % 6.
    // Same slots in both blocks and every step: offsets in a brick and which are in the region
    // are fixed; which are inside the volume is fixed per item.
    const int c = 2 * (lane & 3);
    const float sc0 = s_param[c], sc1 = s_param[c + 1];
    const float sh0 = s_param[8 + c], sh1 = s_param[8 + c + 1];
    uint32_t off[8];
    uint32_t rmask = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int j = i >> 1, m = 16 * wl + (lane >> 2) + 8 * (i & 1);
      const int jr = m / kU9W, jc = m - kU9W * jr;
      const int hh = 2 * jr + (j >> 1) - 1, ww = 2 * jc + (j & 1) - 1;
      const bool in = hh >= 0 && hh < kHaloH && ww >= 0 && ww < kHaloW;
      rmask |= (in ? 1u : 0u) << i;
      off[i] = in ? (c >> 2) * kBrickBytes + (hh * kHaloW + ww) * 16 + (c & 3) * 4 : 0;
    }
    // The epilogue runs after the step's wgmma have retired.  Deferring it past the next step's
    // wgmma, as warpgroup 1 does, keeps the 32 completed accumulators live beside the 48 in
    // flight: ptxas then spills at 96 registers, or needs 112 and leaves one CTA per SM, and
    // both measured slower than waiting here.
    // steps / c0 slots before this item; c0 slot n holds the skip of u11 ring entries 2n, 2n + 1
    uint32_t gin = 0, gc = 0;
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const Chunk t = chunk_of(item);
      uint32_t vmask = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int j = i >> 1, m = 16 * wl + (lane >> 2) + 8 * (i & 1);
        const int jr = m / kU9W, jc = m - kU9W * jr;
        const int oh = t.h0 - 2 + 2 * jr + (j >> 1), ow = t.w0 - 2 + 2 * jc + (j & 1);
        vmask |= (oh >= 0 && oh < p.H && ow >= 0 && ow < p.W ? 1u : 0u) << i;
      }
      vmask &= rmask;
      for (int st = 0; st < t.nsteps; ++st) {
        const uint32_t g = gin + st;
        const int slot = u9_ring.wait(g);
        if (!w_ready) { mbar_wait(bar_w11, 0); w_ready = true; }
        const uint64_t a_s = a_desc0 + ((slot * kU9SlotBytes) >> 4);
        // u9 slice -1 (the first step of a chunk at d0 = 0) is zero fill and feeds only u11
        // slices -3 .. -1, which are never stored or stored as zero: no wgmma for it
        if (t.s0 + st >= 0) {
          wgmma_fence();
#pragma unroll
          for (int tap = 0; tap < 4; ++tap) {
            const int sh = tap >> 1, sw = tap & 1;
#pragma unroll
            for (int k8 = 0; k8 < 2; ++k8) {
              const uint32_t a_off = (2 * k8 * kU9Bytes + (sh * kU9W + sw) * 16) >> 4;
              const uint32_t b_off = (tap * (16 * 96 * 4) + k8 * 2 * 96 * 16) >> 4;
              wgmma_tf32<96>(acc, a_s + a_off, b_desc0 + b_off);
            }
          }
          wgmma_commit();
        }
        wgmma_wait_all();
        u9_ring.release(g);                         // this thread's reads of the slot are done
        // blocks 0 and 1 are complete: u11 slices 2s-1 (pd = 1) and 2s (pd = 0).  Copied out
        // before the per-thread stores (no accumulator register on a divergent path).
        float done[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) done[i] = acc[i];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          acc[i] = acc[32 + i];
          acc[16 + i] = 0.f;
          acc[32 + i] = 0.f;
        }
        if (st == 0) continue;                      // the first step's u11 slices are not used
        const uint32_t gs = gc + st - 1;
        const unsigned char* c0s = smem + kC0Off + c0_ring.wait(gs) * kC0SlotBytes;
#pragma unroll
        for (int k2 = 0; k2 < 2; ++k2) {
          const int us = u_ring.acquire(2 * gs + k2);
          const int od = 2 * (t.s0 + st) - 1 + k2;
          // zero outside the volume (prob's zero padding)
          const uint32_t live = od >= 0 && od < p.D ? vmask : 0u;
          const unsigned char* skip = c0s + k2 * kSliceBytes;
          unsigned char* dst = smem + kUOff + us * kSliceBytes;
          float2 s2[8];
#pragma unroll
          for (int i = 0; i < 8; ++i)
            s2[i] = (live >> i) & 1 ? *reinterpret_cast<const float2*>(skip + off[i])
                                    : make_float2(0.f, 0.f);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            // conv3d_tma2's store2, with the skip from the c0 brick
            const float a0 = done[16 * k2 + 4 * (i >> 1) + 2 * (i & 1)];
            const float a1 = done[16 * k2 + 4 * (i >> 1) + 2 * (i & 1) + 1];
            float v0 = fmaf(a0, sc0, sh0);
            float v1 = fmaf(a1, sc1, sh1);
            v0 = v0 >= 0.f ? v0 : v0 * p.slope;
            v1 = v1 >= 0.f ? v1 : v1 * p.slope;
            v0 += s2[i].x; v1 += s2[i].y;
            const float2 v = (live >> i) & 1 ? make_float2(to_tf32(v0), to_tf32(v1))
                                              : make_float2(0.f, 0.f);
            if ((rmask >> i) & 1) *reinterpret_cast<float2*>(dst + off[i]) = v;
          }
        }
        fence_proxy_async();                        // generic-proxy writes -> prob's wgmma
        u_ring.publish(2 * gs);
        u_ring.publish(2 * gs + 1);
        c0_ring.release(gs);
      }
      gin += t.nsteps;
      gc += t.nsteps - 1;
    }
  } else {
    // ============ warpgroup 1: prob, both 64-row halves of the tile, per u11 slice ============
    constexpr uint32_t a_lbo = kBrickBytes, a_sbo = kHaloW * 16;
    constexpr uint32_t b_lbo = 8 * 16, b_sbo = 128;
    const uint64_t a_desc0 = make_desc(s_u, a_lbo, a_sbo);
    const uint64_t b_desc0 = make_desc(s_base + kWp8Off, b_lbo, b_sbo);
    // column groups 0, 1, 2 = output slices k-2, k-1, k of u11 slice d0-1+k (conv3d_tma.cu)
    float acc0[4], acc1[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    // The completed output slice pend_od of item (pend_b, pend_h0, pend_w0) (< 0: none): its
    // logits are stored while the next u11 slice's wgmma execute.
    float done0[4], done1[4];
    int pend_od = -1, pend_b = 0, pend_h0 = 0, pend_w0 = 0;
    auto store_logits = [&](const float* src, int half) {
      if ((lane & 3) != 0) return;                  // column 0: the only output channel
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = 64 * half + 16 * wl + (lane >> 2) + 8 * h;
        const int oh = pend_h0 + (m >> 3), ow = pend_w0 + (m & 7);
        if (oh >= p.H || ow >= p.W) continue;
        // conv3d_tma's store_slice with Cout = 1, slope 1 (identity) and fp32 output
        p.logits[(((size_t)pend_b * p.D + pend_od) * p.H + oh) * p.W + ow] =
            fmaf(src[2 * h], s_param[16], s_param[24]);
      }
    };
    uint32_t gu = 0;                                // u11 slices before this item
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const Chunk t = chunk_of(item);
      for (int k = 0; k < t.nd + 2; ++k) {
        const uint32_t u = gu + k;
        const int us = u_ring.wait(u);
        if (!w_ready) {
          // the packed image from the unfused layer's, by this warpgroup, for its own wgmma
          mbar_wait(bar_wp, 0);
          const float* src = reinterpret_cast<const float*>(smem + kWpOff);
          float* dst = reinterpret_cast<float*>(smem + kWp8Off);
          for (int i = threadIdx.x - 128; i < kWp8Bytes / 4; i += 128) {
            const int r = i >> 5, n = (i >> 2) & 7;          // r = (kh, kw, cq)
            dst[i] = n < 3 ? src[(r * 24 + 8 * n) * 4 + (i & 3)] : 0.f;
          }
          fence_proxy_async();                      // generic-proxy writes -> wgmma
          asm volatile("bar.sync 1, 128;" ::: "memory");
          w_ready = true;
        }
        const uint64_t a_s = a_desc0 + ((us * kSliceBytes) >> 4);
        // u11 slice -1 (k = 0 at d0 = 0) is zero padding, and the one column group it feeds
        // that is stored (2) starts at +0: without its wgmma that group stays +0
        if (t.d0 - 1 + k >= 0) {
          wgmma_fence();
#pragma unroll
          for (int khw = 0; khw < 9; ++khw) {
            const int kh = khw / 3, kw = khw % 3;
            const uint32_t a_off = ((kh * kHaloW + kw) * 16) >> 4;
            const uint32_t b_off = (khw * (8 * 8 * 4)) >> 4;
            wgmma_tf32<8>(acc0, a_s + a_off, b_desc0 + b_off);
            wgmma_tf32<8>(acc1, a_s + a_off + ((8 * a_sbo) >> 4), b_desc0 + b_off);
          }
          wgmma_commit();
        }
        if (pend_od >= 0) {                         // overlaps this slice's wgmma
          store_logits(done0, 0);
          store_logits(done1, 1);
        }
        wgmma_wait_all();
        u_ring.release(u);
#pragma unroll
        for (int i = 0; i < 4; ++i) { done0[i] = acc0[i]; done1[i] = acc1[i]; }
        // roll the window: columns 1, 2 -> 0, 1 and column 2 = +0.  Fragment: lane 4j holds
        // columns 0, 1 (rows r, r + 8 in registers 0, 1 / 2, 3), lane 4j + 1 columns 2, 3.
        // Selects rather than branches: no accumulator register on a divergent path.
        {
          const bool c01 = (lane & 3) == 0;
          const float z = opaque_zero();
          const float u0 = shfl_down_1(acc0[0]), u2 = shfl_down_1(acc0[2]);
          const float v0 = shfl_down_1(acc1[0]), v2 = shfl_down_1(acc1[2]);
          acc0[0] = c01 ? acc0[1] : z; acc0[2] = c01 ? acc0[3] : z;
          acc0[1] = c01 ? u0 : acc0[1]; acc0[3] = c01 ? u2 : acc0[3];
          acc1[0] = c01 ? acc1[1] : z; acc1[2] = c01 ? acc1[3] : z;
          acc1[1] = c01 ? v0 : acc1[1]; acc1[3] = c01 ? v2 : acc1[3];
        }
        pend_od = k >= 2 ? t.d0 + k - 2 : -1;
        pend_b = t.b; pend_h0 = t.h0; pend_w0 = t.w0;
      }
      gu += t.nd + 2;
    }
    if (pend_od >= 0) {                             // the CTA's last output slice
      store_logits(done0, 0);
      store_logits(done1, 1);
    }
  }
}

static int launch_tail(const TailArgs& a, cudaStream_t st) {
  static_assert(kTotal <= 227 * 1024, "shared memory budget");
  auto kfn = conv3d_tail_kernel;
  static std::atomic<bool> attr_set[kMaxDevices];
  if (int rc = opt_in_smem(kfn, kTotal, attr_set, "conv3d_tail")) return rc;
  Params p;
  p.scale11 = a.scale11; p.shift11 = a.shift11; p.scalep = a.scalep; p.shiftp = a.shiftp;
  p.logits = a.logits; p.slope = a.slope;
  p.B = a.B; p.D = a.D; p.H = a.h; p.W = a.w;
  p.work.tiles_w = (a.w + kTileW - 1) / kTileW;
  p.work.tiles_h = (a.h + kTileH - 1) / kTileH;
  CUtensorMap u9map, c0map;
  if (int rc = input_map(&u9map, a.u9, a.B, a.D / 2, a.h / 2, a.w / 2, 16, kU9W, kU9H, 1, true))
    return rc;
  if (int rc = input_map(&c0map, a.c0, a.B, a.D, a.h, a.w, 8, kHaloW, kHaloH, 1, true)) return rc;
  ImageRef i11, ip;
  if (int rc = conv3d_tma2_conv11_image(a.w11, st, &i11)) return rc;
  if (int rc = conv3d_tma_prob_image(a.wp, st, &ip)) return rc;
  p.img11 = i11.img; p.imgp = ip.img;
  // chunks of dc u9 slices: an item walks dc + 2 u9 slices and 2 dc + 2 u11 slices (the prob
  // halo), and covers 2 dc output slices
  const Sizing z = size_persistent(kfn, kTotal, 1, (long)p.B * p.work.tiles_w * p.work.tiles_h,
                                   p.D / 2, 16, 2, 3);
  p.work.dchunk = 2 * z.dchunk;
  p.work.nchunks = z.nchunks;
  launch_pdl(i11.settled && ip.settled, kfn, z.grid, kConvThreads, kTotal, st, u9map, c0map, p);
  return after_launch("conv3d_tail");
}

// Coverage: (u9 channels, skip channels, output channels) -- CostRegNet's conv11 + prob for
// every input width, since neither depends on the stage's Cin.
struct Shape {
  int cin, cskip, cout;
  TailLauncher run;
};
static const Shape kShapes[] = {{16, 8, 1, launch_tail}};

}  // namespace tail

TailLauncher conv3d_tail_find(int cin, int cskip, int cout) {
  for (const tail::Shape& s : tail::kShapes)
    if (s.cin == cin && s.cskip == cskip && s.cout == cout) return s.run;
  return nullptr;
}

}  // namespace casmvs
