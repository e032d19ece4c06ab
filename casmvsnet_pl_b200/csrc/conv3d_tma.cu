// K2 (tensor-core variant, TMA producer) — 3x3x3 stride-1 convolution as an im2col-free
// implicit GEMM on wgmma (tf32 operands from shared memory, fp32 accumulators in registers)
// with the norm-act (+skip) epilogue fused.  sm_90a.
//
// Replaces (reference): ConvBnReLU3D (models/modules.py:21-31) and the `prob` head
// (models/mvsnet.py:89,103) for the stride-1 layers of CostRegNet (conv0, conv2, conv4, conv6,
// prob), and the 1x3x3 planar convolutions of FeatureNet.
//
// The GEMM: M = 128 voxels = 8(w) x 16(h) of one depth slice, K = Cin per tap, N = 3 x GW (the
// three kd taps share one A operand: an input slice feeds three output slices in ONE wgmma).
// The input brick of a depth slice (18 x 10 voxels with halo) is brought in by Cin/4 TMA tiled
// loads (cp.async.bulk.tensor.5d over x viewed as {C, W, H, D, B}, a box of 4 channels each, or,
// for x blocked by channel quads, as {4W, H, D, C/4, B}, a box of one quad's 160-byte rows;
// out-of-bounds elements are zero-filled by the TMA unit = the conv's zero padding, in all
// three spatial dimensions).  Each load writes one [18][10][4 channels] brick: 16 bytes per
// voxel, so 8 consecutive voxels of a brick row are one 128-byte wgmma core matrix and the A
// operand of tap (kh,kw) is a SHIFTED VIEW of the bricks: descriptor start = brick +
// (kh*10 + kw)*16 B, K direction = next brick (LBO), next 8-voxel row group = next brick row
// (SBO = 160 B).  No swizzle, so any 16-byte-aligned start address is a valid view.
//
// Persistent CTAs, 9 warps: two consumer warpgroups (rows 0-63 and 64-127 of the tile) and a
// TMA producer warp.  Ring full barriers are armed with expect_tx and completed by the TMA
// unit; ring empty barriers by the 256 consumer threads once their wgmma have retired.  The
// accumulator of one input slice covers output slices it-2, it-1, it (column groups 0, 1, 2);
// after the slice, group 0 is complete: it is copied out, the window rolls, the next slice's
// wgmma are issued and group 0's epilogue runs while they execute.  N = 3 x GW with GW = 8 for
// Cout <= 8 (conv0, prob, FeatureNet's last smoothing layer), else 16 or 32.
#include <cudaTypedefs.h>

#include "common.cuh"
#include "tc_common.cuh"
#include <string.h>
#include <mutex>

#include "tma_common.cuh"

namespace casmvs {

namespace tma {

using namespace tc;

struct Params {
  const float* bimg;    // pre-built B operand image [chunk][kh][kw][CIN/4][3*GW][4] (tf32-rounded)
  const float* scale;   // [Cout] or null
  const float* shift;   // [Cout] or null
  const float* skip;    // (B,D,H,W,Cout) or null
  float* y;             // (B,D,H,W,Cout)
  float slope;
  int B, D, H, W, Cout;   // Cout = channels handled by one CTA (<= GW)
  int cout_total;         // channel count of the output tensor; blockIdx.y selects the chunk
  Work work;
  int round_out;        // round the stored activations to tf32 (unbiased next-layer operand)
  int x_blocked;        // x stored blocked by channel quads (input_map); else channels-last
  int y_blocked;        // y and skip stored blocked by channel quads; else channels-last
};

template <int CIN, int GW, int SLOTS_>
struct Smem {
  static constexpr int SLOTS = SLOTS_;
  static constexpr int CQ = CIN / 4;                                // bricks (4 channels) per slice
  static constexpr int kBrickData = kHaloH * kHaloW * 16;           // bytes one TMA load writes
  static constexpr int kBrickBytes = (kBrickData + 127) / 128 * 128;
  static constexpr int kSlotBytes = CQ * kBrickBytes;
  static constexpr int kWBytes = 9 * CIN * 3 * GW * 4;              // [kh][kw][cq][3*GW][4]
  static constexpr int kRingOff = 0;
  static constexpr int kWOff = SLOTS * kSlotBytes;
  static constexpr int kParamOff = kWOff + kWBytes;                 // scale/shift [2][GW]
  static constexpr int kBarOff = kParamOff + 2 * GW * 4;
  // barriers: full[8] @0, empty[8] @64, weight image @128
  static constexpr int kTotal = kBarOff + 192 + 1024;               // + alignment slack
};

// Epilogue of one output slice from the accumulator columns [OFF, OFF + GW) of this thread's
// fragment: scale/shift, leaky ReLU, optional skip, optional tf32 rounding, channels-last or
// blocked store (p.y_blocked).
template <int GW, int OFF, bool PLANAR>
__device__ __forceinline__ void store_slice(const float* acc, const Params& p, const float* s_param,
                                            int b, int od, int h0, int w0, int row0, int wl,
                                            int lane, int co_base) {
  for_each_pair<OFF, GW>(acc, wl, lane, [&](int r, int c, float a0, float a1) {
    const int m = row0 + r;
    const int oh = h0 + (m >> 3), ow = w0 + (m & 7);
    if (oh >= p.H || ow >= p.W || c >= p.Cout) return;
    const size_t o =
        vol_offset(!PLANAR && p.y_blocked, b, od, oh, ow, co_base + c, p.D, p.H, p.W, p.cout_total);
    float v0 = fmaf(a0, s_param[c], s_param[GW + c]);
    float v1 = fmaf(a1, s_param[c + 1], s_param[GW + c + 1]);
    v0 = v0 >= 0.f ? v0 : v0 * p.slope;
    v1 = v1 >= 0.f ? v1 : v1 * p.slope;
    if (c + 1 < p.Cout && (p.cout_total & 1) == 0) {
      if (p.skip) {
        const float2 s2 = __ldg(reinterpret_cast<const float2*>(p.skip + o));
        v0 += s2.x; v1 += s2.y;
      }
      if (p.round_out) { v0 = to_tf32(v0); v1 = to_tf32(v1); }
      *reinterpret_cast<float2*>(p.y + o) = make_float2(v0, v1);
    } else {
      if (p.skip) v0 += __ldg(p.skip + o);
      p.y[o] = p.round_out ? to_tf32(v0) : v0;
      if (c + 1 < p.Cout) {
        if (p.skip) v1 += __ldg(p.skip + o + 1);
        p.y[o + 1] = p.round_out ? to_tf32(v1) : v1;
      }
    }
  });
}

template <int CIN, int GW, int SLOTS_, bool PLANAR>
__global__ void __launch_bounds__(kConvThreads, 1)
conv3d_tma_kernel(const __grid_constant__ CUtensorMap xmap, const Params p) {
  using S = Smem<CIN, GW, SLOTS_>;
  constexpr int SLOTS = S::SLOTS;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem;
  const uint32_t s_base = smem_align_1024(smem_raw, &smem);
  const uint32_t s_ring = s_base + S::kRingOff, s_w = s_base + S::kWOff,
                 s_bar = s_base + S::kBarOff;
  float* s_param = reinterpret_cast<float*>(smem + S::kParamOff);
  const Ring<SLOTS> ring{s_bar, s_bar + 64};
  const uint32_t bar_w = s_bar + 128;

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int total_items = p.B * p.work.nchunks * p.work.tiles_h * p.work.tiles_w;

  // ---- one-time setup ----
  {
    const int t = threadIdx.x;
    ring.init(t, 1, kConsumerThreads);
    if (t == 2 * SLOTS) mbar_init(bar_w, 1);
    if (t <= 2 * SLOTS) fence_barrier_init();
  }
  const int co_base = blockIdx.y * p.Cout;
  stage_scale_shift<GW>(s_param, p.scale, p.shift, co_base, p.Cout);
  end_prologue(ImageCopy{s_w, p.bimg + (size_t)blockIdx.y * (S::kWBytes / 4), S::kWBytes, bar_w});
  bool w_ready = false;                             // consumers: weight image has landed
  uint32_t gs = 0;                                  // slices processed before this item (all roles)
  // consumers: the accumulator, column groups 0, 1, 2 = output slices it-2, it-1, it (planar:
  // one group, output slice it); and the completed output slice whose epilogue is pending
  // (od < 0: none).  Both carry over into the CTA's next item.
  float acc[(PLANAR ? 1 : 3) * GW / 2];
#pragma unroll
  for (int i = 0; i < (PLANAR ? 1 : 3) * GW / 2; ++i) acc[i] = 0.f;
  float done[GW / 2];
  int pend_od = -1, pend_b = 0, pend_h0 = 0, pend_w0 = 0;
  const int wg = warp >> 2, wl = warp & 3;
  const int row0 = 64 * wg;                         // consumers: first GEMM row of the warpgroup
  for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
    const Item t = decode_item(item, p.work);
    const int b = t.b, h0 = t.h0, w0 = t.w0;
    const int d0 = t.chunk * p.work.dchunk, d1 = min(p.D, d0 + p.work.dchunk);
    const int nd = d1 - d0;
    const int halo = PLANAR ? 0 : 1;
    const int nslices = nd + 2 * halo;              // input slices d0-halo .. d1-1+halo

    if (warp == kProdWarp) {
      // ===================== producer: Cin/4 TMA loads per slice =====================
      if (lane == 0) {
        for (int it = 0; it < nslices; ++it) {
          const uint32_t g = gs + it;
          const uint32_t dst = s_ring + ring.acquire(g) * S::kSlotBytes, full = ring.full_bar(g);
          mbar_expect_tx(full, S::CQ * S::kBrickData);
#pragma unroll
          for (int q = 0; q < S::CQ; ++q) {
            const Coords5 k = brick_coords(!PLANAR && p.x_blocked, q, w0 - 1, h0 - 1,
                                           d0 - halo + it, b);
            tma_load_5d(dst + q * S::kBrickBytes, &xmap, full, k.c[0], k.c[1], k.c[2], k.c[3],
                        k.c[4]);
          }
        }
      }
      __syncwarp();
    } else {
      // == consumer warpgroups: wgmma into registers; the previous output slice's epilogue ==
      // == runs while they execute                                                        ==
      constexpr uint32_t a_lbo = S::kBrickBytes, a_sbo = kHaloW * 16;   // 8-voxel group stride
      constexpr uint32_t b_lbo = 3 * GW * 16, b_sbo = 128;
      const uint64_t a_desc0 = make_desc(s_ring + 8 * wg * a_sbo, a_lbo, a_sbo);
      const uint64_t b_desc0 = make_desc(s_w, b_lbo, b_sbo);
      for (int it = 0; it < nslices; ++it) {
        const uint32_t g = gs + it;
        const int slot = ring.wait(g);
        if (!w_ready) { mbar_wait(bar_w, 0); w_ready = true; }
        const uint64_t a_s = a_desc0 + ((slot * S::kSlotBytes) >> 4);
        wgmma_fence();
#pragma unroll
        for (int khw = 0; khw < 9; ++khw) {
          const int kh = khw / 3, kw = khw % 3;
#pragma unroll
          for (int k8 = 0; k8 < CIN / 8; ++k8) {
            const uint32_t a_off = ((kh * kHaloW + kw) * 16 + 2 * k8 * S::kBrickBytes) >> 4;
            const uint32_t b_off = (khw * (CIN * 3 * GW * 4) + k8 * 2 * 3 * GW * 16) >> 4;
            if constexpr (PLANAR)   // kd = 1 only: B column group 1
              wgmma_tf32<GW>(acc, a_s + a_off, b_desc0 + b_off + ((GW * 16) >> 4));
            else
              wgmma_tf32<3 * GW>(acc, a_s + a_off, b_desc0 + b_off);
          }
        }
        wgmma_commit();
        // the epilogue of the output slice completed by the previous input slice (possibly
        // the last one of the previous item) overlaps this slice's wgmma
        if (pend_od >= 0)
          store_slice<GW, 0, PLANAR>(done, p, s_param, pend_b, pend_od, pend_h0, pend_w0, row0, wl,
                                     lane, co_base);
        wgmma_wait_all();
        ring.release(g);                            // this thread's reads of the slot are done
        // output slice of column group 0: `it` when planar, else it - 2 (complete after its
        // third input slice).  Group 0 is copied out before the (per-thread) stores so that no
        // accumulator register is touched on a divergent path: that would make ptxas serialize
        // the wgmma of the next slice.  At an item boundary groups 0 and 1 hold the output
        // slices -2 and -1 of the next item, which are never stored.
#pragma unroll
        for (int i = 0; i < GW / 2; ++i) done[i] = acc[i];
        if constexpr (PLANAR) {
#pragma unroll
          for (int i = 0; i < GW / 2; ++i) acc[i] = 0.f;
        } else {
#pragma unroll
          for (int i = 0; i < GW; ++i) acc[i] = acc[i + GW / 2];   // groups 1, 2 -> 0, 1
#pragma unroll
          for (int i = 0; i < GW / 2; ++i) acc[GW + i] = 0.f;
        }
        const int j = PLANAR ? it : it - 2;
        pend_od = (j >= 0 && j < nd) ? d0 + j : -1;
        pend_b = b; pend_h0 = h0; pend_w0 = w0;
      }
    }
    gs += nslices;
  }
  if (pend_od >= 0)                                 // consumers: the CTA's last output slice
    store_slice<GW, 0, PLANAR>(done, p, s_param, pend_b, pend_od, pend_h0, pend_w0, row0, wl, lane,
                               co_base);
}

// ---- host side ----

int encode_map(const MapDesc& d, CUtensorMap* out) {
  static_assert(sizeof(MapDesc) == 128, "MapDesc is compared bytewise: no padding");
  static const PFN_cuTensorMapEncodeTiled_v12000 enc = [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    return cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) ==
                   cudaSuccess && q == cudaDriverEntryPointSuccess
               ? reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr)
               : nullptr;
  }();
  struct Entry { MapDesc d; CUtensorMap map; };
  static Entry memo[128];
  static int memo_n = 0, memo_next = 0;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  for (int i = 0; i < memo_n; ++i) {
    if (memcmp(&memo[i].d, &d, sizeof(MapDesc)) == 0) {
      *out = memo[i].map;
      return 0;
    }
  }
  if (!enc) { set_error("tma: cuTensorMapEncodeTiled is not available"); return -2; }
  const CUtensorMapSwizzle sw = d.swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : d.swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : d.swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                        : CU_TENSOR_MAP_SWIZZLE_NONE;
  const CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)d.rank,
                         const_cast<void*>(d.base), d.dims, d.strides_bytes, d.box, d.elem_strides,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("tma: cuTensorMapEncodeTiled failed (%d), rank %d, dims %llu %llu %llu %llu %llu",
              (int)r, d.rank, (unsigned long long)d.dims[0], (unsigned long long)d.dims[1],
              (unsigned long long)d.dims[2], (unsigned long long)d.dims[3],
              (unsigned long long)d.dims[4]);
    return -2;
  }
  memo[memo_next] = Entry{d, *out};
  memo_next = (memo_next + 1) % 128;
  if (memo_n < 128) ++memo_n;
  return 0;
}

int input_map(CUtensorMap* out, const float* x, int B, int D, int H, int W, int C, int box_w,
              int box_h, int stride_w, bool blocked) {
  if (blocked && stride_w != 1) {
    set_error("tma: a blocked input map walks W with stride 1 (got %d)", stride_w);
    return -2;
  }
  const uint64_t c = C, w = W, h = H, dp = D, b = B, vox = dp * h * w;
  const uint32_t bw = box_w, bh = box_h, sw = stride_w;
  const MapDesc d =
      !blocked ? MapDesc{x, 5, 0, {c, w, h, dp, b}, {4 * c, 4 * c * w, 4 * c * w * h, 4 * c * vox},
                         {4, bw, bh, 1, 1}, {1, sw, 1, 1, 1}}
               : MapDesc{x, 5, 0, {4 * w, h, dp, c / 4, b}, {16 * w, 16 * w * h, 16 * vox, 4 * c * vox},
                         {4 * bw, bh, 1, 1, 1}, {1, 1, 1, 1, 1}};
  return encode_map(d, out);
}

// B operand image of the stride-1 kernels: [chunk][kh][kw][CIN/4][3*GW][4], column group g
// holds the weights of kd = 2 - g, tf32-rounded (to nearest), zero rows for co >= chunk.  One
// image per Cout chunk (chunk = blockIdx.y of the conv kernel), `chunk` channels each.
__global__ void build_image_kernel(const float* __restrict__ wpk, float* __restrict__ img,
                                   int CIN, int GW, int chunk, int cout_total) {
  const int CQ = CIN / 4;
  const int per = 9 * CIN * 3 * GW;
  const int total = per * (cout_total / chunk);
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    const int ck = t / per, i = t - ck * per;
    const int j = i & 3;
    const int n = (i >> 2) % (3 * GW);
    const int r = (i >> 2) / (3 * GW);    // (kh*3+kw)*CQ + cq
    const int cq = r % CQ, khw = r / CQ;
    const int g = n / GW, co = n % GW;
    const int kd = 2 - g;
    const int ci = cq * 4 + j;
    float v = 0.f;
    if (co < chunk)
      v = to_tf32(__ldg(wpk + ((size_t)(kd * 9 + khw) * CIN + ci) * cout_total + ck * chunk + co));
    img[t] = v;
  }
}

// The B operand image of a layer (nco chunks of GW columns, `cout` of them used).
template <int CIN, int GW>
static int stride1_image(const float* wpk, int cout, int cout_total, int nco, cudaStream_t st,
                         ImageRef* ir) {
  return cached_image(wpk, 1000 + CIN * 100 + GW, (size_t)Smem<CIN, GW, 1>::kWBytes * nco, st, ir,
                      "conv3d_tma/build_image", [&](float* img) {
                        build_image_kernel<<<64, 256, 0, st>>>(wpk, img, CIN, GW, cout, cout_total);
                      });
}

// One CTA computes GW output columns (Cout <= GW, or a GW-channel slice of a wider Cout).
template <int CIN, int GW, int SLOTS, bool PLANAR>
static int launch(const ConvArgs& a, cudaStream_t st) {
  using S = Smem<CIN, GW, SLOTS>;
  static_assert(S::kTotal <= 227 * 1024, "shared memory budget");
  auto kfn = conv3d_tma_kernel<CIN, GW, SLOTS, PLANAR>;
  static std::atomic<bool> attr_set[kMaxDevices];
  if (int rc = opt_in_smem(kfn, S::kTotal, attr_set, "conv3d_tma")) return rc;
  Params p;
  p.scale = a.scale; p.shift = a.shift; p.skip = a.skip; p.y = a.y;
  p.slope = a.slope; p.B = a.B; p.D = a.D; p.H = a.h; p.W = a.w;
  p.Cout = a.Cout < GW ? a.Cout : GW; p.cout_total = a.Cout;
  p.work.tiles_w = (a.w + tc::kTileW - 1) / tc::kTileW;
  p.work.tiles_h = (a.h + tc::kTileH - 1) / tc::kTileH;
  p.x_blocked = (a.layout & kLayoutXBlocked) ? 1 : 0;
  p.y_blocked = (a.layout & kLayoutYBlocked) ? 1 : 0;
  p.round_out = a.round_out;
  CUtensorMap map;
  if (int rc = input_map(&map, a.x, p.B, p.D, p.H, p.W, CIN, kHaloW, kHaloH, 1, p.x_blocked))
    return rc;
  const int nco = p.cout_total / p.Cout;
  const Sizing z = size_persistent(kfn, S::kTotal, nco, (long)p.B * p.work.tiles_w * p.work.tiles_h,
                                   p.D, 32, 1, PLANAR ? 0 : 2);
  p.work.dchunk = z.dchunk;
  p.work.nchunks = z.nchunks;
  ImageRef ir;
  if (int rc = stride1_image<CIN, GW>(a.wpk, p.Cout, p.cout_total, nco, st, &ir)) return rc;
  p.bimg = ir.img;
  launch_pdl(ir.settled, kfn, z.grid, kConvThreads, S::kTotal, st, map, p);
  return after_launch("conv3d_tma");
}

// Coverage: the stride-1 and planar layer shapes this kernel is instantiated for.  Cout in
// [cout_lo, cout_hi] runs on GW output columns; conv6 (64 -> 64) as four 16-column slices.
struct Shape {
  int cin, cout_lo, cout_hi;
  ConvLauncher conv, planar;
};
#define S1(CI, LO, HI, GW, SL) {CI, LO, HI, launch<CI, GW, SL, false>, launch<CI, GW, SL, true>}
static const Shape kShapes[] = {
    S1(8, 1, 8, 8, 4),    S1(8, 17, 32, 32, 4),
    S1(16, 1, 8, 8, 4),   S1(16, 9, 16, 16, 4),  S1(16, 17, 32, 32, 4),
    S1(32, 1, 8, 8, 4),   S1(32, 9, 16, 16, 4),  S1(32, 17, 32, 32, 4),
    S1(64, 64, 64, 16, 2),
};
#undef S1

}  // namespace tma

ConvLauncher conv3d_tma_find(int Cin, int Cout, int kind, int stride) {
  if ((kind != CASMVS_CONV && kind != CASMVS_CONV_PLANAR) || stride != 1) return nullptr;
  for (const tma::Shape& s : tma::kShapes)
    if (s.cin == Cin && s.cout_lo <= Cout && Cout <= s.cout_hi)
      return kind == CASMVS_CONV_PLANAR ? s.planar : s.conv;
  return nullptr;
}

int conv3d_tma_prob_image(const float* wpk, cudaStream_t st, tc::ImageRef* ir) {
  return tma::stride1_image<8, 8>(wpk, 1, 1, 1, st, ir);
}

}  // namespace casmvs
