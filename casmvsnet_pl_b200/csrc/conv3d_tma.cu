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
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"
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
  int tiles_w, tiles_h, nchunks, dchunk;
  int round_out;        // round the stored activations to tf32 (unbiased next-layer operand)
  int planar;           // 1x3x3 kernel: input slice s feeds output slice s only (kd = 1)
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
  const uint32_t s_raw = smem_u32(smem_raw);
  const uint32_t s_base = (s_raw + 1023u) & ~1023u;
  unsigned char* smem = smem_raw + (s_base - s_raw);
  const uint32_t s_ring = s_base + S::kRingOff, s_w = s_base + S::kWOff,
                 s_bar = s_base + S::kBarOff;
  float* s_param = reinterpret_cast<float*>(smem + S::kParamOff);
  const uint32_t bar_full = s_bar, bar_empty = s_bar + 64, bar_w = s_bar + 128;

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int total_items = p.B * p.nchunks * p.tiles_h * p.tiles_w;

  // ---- one-time setup ----
  {
    const int t = threadIdx.x;
    if (t < SLOTS) mbar_init(bar_full + 8 * t, 1);
    else if (t < 2 * SLOTS) mbar_init(bar_empty + 8 * (t - SLOTS), kConsumerThreads);
    else if (t == 2 * SLOTS) mbar_init(bar_w, 1);
    if (t <= 2 * SLOTS) fence_barrier_init();
  }
  const int co_base = blockIdx.y * p.Cout;
  for (int i = threadIdx.x; i < GW; i += kConvThreads) {
    s_param[i] = (i < p.Cout) ? (p.scale ? __ldg(p.scale + co_base + i) : 1.f) : 0.f;
    s_param[GW + i] = (i < p.Cout) ? (p.shift ? __ldg(p.shift + co_base + i) : 0.f) : 0.f;
  }
  fence_proxy_async();
  __syncthreads();
  if (threadIdx.x == 0) load_image_bulk(s_w, p.bimg + (size_t)blockIdx.y * (S::kWBytes / 4), S::kWBytes, bar_w);

  // nothing above depends on the previous kernel of the stream (see tma_common.cuh)
  tma::pdl_trigger();
  tma::pdl_wait();
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
  for (int item0 = blockIdx.x; item0 < total_items; item0 += gridDim.x) {
    int item = item0;
    const int tw = item % p.tiles_w; item /= p.tiles_w;
    const int th = item % p.tiles_h; item /= p.tiles_h;
    const int ck = item % p.nchunks;
    const int b = item / p.nchunks;
    const int w0 = tw * kTileW, h0 = th * kTileH;
    const int d0 = ck * p.dchunk, d1 = min(p.D, d0 + p.dchunk);
    const int nd = d1 - d0;
    const int halo = PLANAR ? 0 : 1;
    const int nslices = nd + 2 * halo;              // input slices d0-halo .. d1-1+halo

    if (warp == kProdWarp) {
      // ===================== producer: Cin/4 TMA loads per slice =====================
      if (lane == 0) {
        for (int it = 0; it < nslices; ++it) {
          const uint32_t g = gs + it;
          const int slot = g % SLOTS;
          if (g >= (uint32_t)SLOTS) mbar_wait(bar_empty + 8 * slot, ((g / SLOTS) - 1) & 1);
          const uint32_t dst = s_ring + slot * S::kSlotBytes;
          mbar_expect_tx(bar_full + 8 * slot, S::CQ * S::kBrickData);
#pragma unroll
          for (int q = 0; q < S::CQ; ++q) {
            const Coords5 k = brick_coords(!PLANAR && p.x_blocked, 1, S::CQ, q, w0 - 1, h0 - 1,
                                           d0 - halo + it, b);
            tma_load_5d(dst + q * S::kBrickBytes, &xmap, bar_full + 8 * slot, k.c[0], k.c[1],
                        k.c[2], k.c[3], k.c[4]);
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
        mbar_wait(bar_full + 8 * (g % SLOTS), (g / SLOTS) & 1);
        if (!w_ready) { mbar_wait(bar_w, 0); w_ready = true; }
        const uint64_t a_s = a_desc0 + (((g % SLOTS) * S::kSlotBytes) >> 4);
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
        mbar_arrive(bar_empty + 8 * (g % SLOTS));   // this thread's reads of the slot are done
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

static PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) ==
            cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  }
  return fn;
}

// Generic tiled-map encoder for other kernels of the library (K1's feature boxes): fp32
// elements, rank <= 5, zero fill out of bounds.  0 on success.
int encode_tiled(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  auto enc = encode_fn();
  if (!enc) { set_error("tma: cuTensorMapEncodeTiled is not available"); return -2; }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                      : CU_TENSOR_MAP_SWIZZLE_NONE;
  const CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank,
                         const_cast<void*>(base), gdim, gstr, bx, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("tma: cuTensorMapEncodeTiled failed (%d), rank %d", (int)r, rank);
    return -2;
  }
  return 0;
}

// Tensor maps are pure functions of (pointer, shape, box): memoised, since inference calls
// every layer with the same workspace pointers each step.
struct MapEntry { const void* x; int B, D, H, W, C, CB, bw, bh, sw, blk; CUtensorMap map; };
static MapEntry g_maps[128];
static int g_maps_n = 0, g_maps_next = 0;
static std::mutex g_maps_mu;

const CUtensorMap* input_map(const float* x, int B, int D, int H, int W, int C, int CB, int box_w,
                             int box_h, int stride_w, bool blocked) {
  // the returned map is a per-thread copy: ring slots may be recycled by other threads
  static thread_local CUtensorMap t_ret;
  const int blk = blocked ? 1 : 0;
  std::lock_guard<std::mutex> lock(g_maps_mu);
  for (int i = 0; i < g_maps_n; ++i) {
    const MapEntry& e = g_maps[i];
    if (e.x == x && e.B == B && e.D == D && e.H == H && e.W == W && e.C == C && e.CB == CB &&
        e.bw == box_w && e.bh == box_h && e.sw == stride_w && e.blk == blk) {
      t_ret = e.map;
      return &t_ret;
    }
  }
  auto enc = encode_fn();
  if (!enc) { set_error("conv3d_tma: cuTensorMapEncodeTiled is not available"); return nullptr; }
  MapEntry& e = g_maps[g_maps_next];
  g_maps_next = (g_maps_next + 1) % 128;
  if (g_maps_n < 128) ++g_maps_n;
  const cuuint64_t vox = (cuuint64_t)D * H * W;      // voxels per channel plane
  // channels-last (B,D,H,W,C) as {C, W, H, D, B}, box {CB, box_w, box_h, 1, 1}
  cuuint64_t gdim[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)D, (cuuint64_t)B};
  cuuint64_t gstr[4] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4,
                        vox * C * 4};
  cuuint32_t box[5] = {(cuuint32_t)CB, (cuuint32_t)box_w, (cuuint32_t)box_h, 1, 1};
  cuuint32_t estr[5] = {1, (cuuint32_t)stride_w, 1, 1, 1};
  if (blocked && stride_w == 1) {
    // blocked (B,C/4,D,H,W,4) as {4W, H, D, C/4, B}: the quad folded into the inner dimension,
    // box {4 box_w, box_h, 1, 1, 1}: one brick row is 16 box_w contiguous bytes
    const cuuint64_t d2[5] = {4 * (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)D, (cuuint64_t)C / 4,
                              (cuuint64_t)B};
    const cuuint64_t s2[4] = {(cuuint64_t)W * 16, (cuuint64_t)H * W * 16, vox * 16, vox * C * 4};
    const cuuint32_t b2[5] = {4 * (cuuint32_t)box_w, (cuuint32_t)box_h, 1, 1, 1};
    for (int i = 0; i < 5; ++i) { gdim[i] = d2[i]; box[i] = b2[i]; estr[i] = 1; }
    for (int i = 0; i < 4; ++i) gstr[i] = s2[i];
  } else if (blocked) {
    // blocked, W walked with element stride 2: {4, W, H, D, C/4 * B}, box {4, box_w, box_h, 1, 1}
    const cuuint64_t d2[5] = {4, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)D,
                              (cuuint64_t)C / 4 * B};
    const cuuint64_t s2[4] = {16, (cuuint64_t)W * 16, (cuuint64_t)H * W * 16, vox * 16};
    for (int i = 0; i < 5; ++i) gdim[i] = d2[i];
    for (int i = 0; i < 4; ++i) gstr[i] = s2[i];
    box[0] = 4;
  }
  const CUtensorMapSwizzle sw = CB * 4 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : CB * 4 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : CB * 4 == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                               : CU_TENSOR_MAP_SWIZZLE_NONE;
  const CUresult r = enc(&e.map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(x), gdim,
                         gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    e.x = nullptr;
    set_error("conv3d_tma: cuTensorMapEncodeTiled failed (%d) for C=%d W=%d H=%d D=%d B=%d",
              (int)r, C, W, H, D, B);
    return nullptr;
  }
  e.x = x; e.B = B; e.D = D; e.H = H; e.W = W; e.C = C; e.CB = CB; e.bw = box_w; e.bh = box_h;
  e.sw = stride_w; e.blk = blk;
  t_ret = e.map;
  return &t_ret;
}


template <int CIN, int GW, int SLOTS, bool PLANAR>
static int launch(const float* x, const float* wpk, Params p, cudaStream_t st) {
  using S = Smem<CIN, GW, SLOTS>;
  static_assert(S::kTotal <= 227 * 1024, "shared memory budget");
  auto kfn = conv3d_tma_kernel<CIN, GW, SLOTS, PLANAR>;
  static std::atomic<bool> attr_set[kMaxDevices];
  if (int rc = opt_in_smem(kfn, S::kTotal, attr_set, "conv3d_tma")) return rc;
  const CUtensorMap* map = input_map(x, p.B, p.D, p.H, p.W, CIN, 4, kHaloW, kHaloH, 1, p.x_blocked);
  if (!map) return -2;
  static int dchunk_env = -1;
  if (dchunk_env < 0) {
    const char* d = getenv("CASMVS_TMA_DCHUNK");
    dchunk_env = d ? atoi(d) : 0;
  }
  const int per_sm = resident_per_sm(kfn, kConvThreads, S::kTotal);
  const int nco = p.cout_total / p.Cout;
  const int cap = 32;
  const long cols = (long)p.B * p.tiles_w * p.tiles_h;
  int dchunk = pick_dchunk(p.D, cap, cols, (long)num_sms() * per_sm / nco, 1, p.planar ? 0 : 2);
  if (dchunk_env > 0 && dchunk_env <= cap) dchunk = dchunk_env < p.D ? dchunk_env : p.D;
  p.dchunk = dchunk;
  p.nchunks = (p.D + dchunk - 1) / dchunk;
  const ImageRef ir = image_cache_get(wpk, 1000 + CIN * 100 + GW, (size_t)S::kWBytes * nco, st);
  if (!ir.img) return -2;
  if (!ir.hit) {
    if (int rc = build_stride1_image(wpk, ir.img, CIN, GW, p.Cout, p.cout_total, st)) return rc;
    image_cache_built(ir.img, st);
  }
  p.bimg = ir.img;
  const long items = (long)p.B * p.nchunks * p.tiles_h * p.tiles_w;
  int resident = num_sms() * per_sm / nco;
  if (resident < 1) resident = 1;
  const long gx = items < resident ? items : resident;
  launch_pdl(ir.settled, kfn, dim3((unsigned)gx, (unsigned)nco), kConvThreads, S::kTotal, st, *map, p);
  return after_launch("conv3d_tma");
}

}  // namespace tma

// CASMVS_TMA (default 1): 0 leaves every layer to the other kernels.
bool conv3d_tma_enabled() {
  static const int enabled = [] {
    const char* e = getenv("CASMVS_TMA");
    return e ? atoi(e) : 1;
  }();
  return enabled != 0;
}

// Returns 0 when handled, 1 when the layer shape is left to the other kernels.
int conv3d_tma(const float* x, const float* wpk, const float* scale, const float* shift,
               float slope, const float* skip, float* y, int B, int Cin, int Cout, int D, int h,
               int w, int kind, int stride, int precision_flags, int layout, cudaStream_t st) {
  const int precision = precision_flags & 0xff;
  static const int round_out = [] {
    const char* s = getenv("CASMVS_TC_ROUND");
    return s ? atoi(s) : 1;
  }();
  if (!conv3d_tma_enabled() || precision != CASMVS_TF32) return 1;
  if ((kind != CASMVS_CONV && kind != CASMVS_CONV_PLANAR) || stride != 1) return 1;
  if (kind == CASMVS_CONV_PLANAR && layout != 0) return 1;   // planar layers are channels-last only
  const bool deep = Cin == 64 && Cout == 64;          // conv6: 16-channel Cout slices
  if (!deep && (!(Cin == 8 || Cin == 16 || Cin == 32) || Cout > 32)) return 1;
  // the TMA global strides must be multiples of 16 B and the base 16 B aligned
  if ((reinterpret_cast<uintptr_t>(x) & 15) != 0) return 1;
  tma::Params p;
  p.scale = scale; p.shift = shift; p.skip = skip; p.y = y;
  p.slope = slope; p.B = B; p.D = D; p.H = h; p.W = w;
  p.Cout = deep ? 16 : Cout; p.cout_total = Cout;
  p.tiles_w = (w + tc::kTileW - 1) / tc::kTileW;
  p.tiles_h = (h + tc::kTileH - 1) / tc::kTileH;
  const int npad = p.Cout <= 8 ? 8 : p.Cout <= 16 ? 16 : 32;
  p.planar = kind == CASMVS_CONV_PLANAR ? 1 : 0;
  p.x_blocked = (layout & kLayoutXBlocked) ? 1 : 0;
  p.y_blocked = (layout & kLayoutYBlocked) ? 1 : 0;
  // the prob head feeds the softmax: keep fp32; callers can ask for unrounded outputs
  p.round_out = (round_out && Cout > 1 && !(precision_flags & CASMVS_KEEP_FP32_OUT)) ? 1 : 0;
#define TMA_CASE(CI, NP, SL)                                                    \
  if (Cin == CI && npad == NP)                                                  \
    return p.planar ? tma::launch<CI, NP, SL, true>(x, wpk, p, st)              \
                    : tma::launch<CI, NP, SL, false>(x, wpk, p, st);
  TMA_CASE(8, 8, 4) TMA_CASE(8, 32, 4) TMA_CASE(16, 8, 4) TMA_CASE(16, 16, 4)
  TMA_CASE(16, 32, 4) TMA_CASE(32, 8, 4) TMA_CASE(32, 16, 4) TMA_CASE(32, 32, 4)
  TMA_CASE(64, 16, 2)
#undef TMA_CASE
  return 1;
}

}  // namespace casmvs
