// K2 (tensor-core variant, TMA producer, part 2) — the stride-2 convolutions (conv1, conv3,
// conv5) and the transposed convolutions (conv7, conv9, conv11) of CostRegNet, and the 5x5
// stride-2 Conv2d layers of FeatureNet, on wgmma (tf32, fp32 accumulators in registers).
// The GEMMs ("resident bricks + shifted-view descriptors", see conv3d_tma.cu):
//   MODE_S2 (stride 2): M = 8(w) x 16(h) OUTPUT voxels of one output slice od.  Input row
//     ih = 2*oh + kh - 1 => consecutive GEMM row groups are two brick rows apart; input column
//     iw = 2*ow + kw - 1 => even and odd columns are separate planes so that 8 consecutive ow are
//     again adjacent.  Odd input slices (s = 2a+1) feed outputs a (kd=2) and a+1 (kd=0) in ONE
//     wgmma of N = 2*GW; even slices feed output a (kd=1).
//   MODE_T (transposed, output = 2x input): M = 8 x 16 INPUT voxels j of one input slice.
//     Output voxel o = 2j + p (p in {0,1}^3, 8 parity classes); class p reads input j + s with
//     tap k:  p=0 -> (s=0,k=1);  p=1 -> (s=0,k=2) and (s=1,k=0).  For each of the 4 in-plane
//     shifts (sh,sw) the A view is shared by every (class, kd) it reaches, so one wgmma of
//     N = 12*Cout covers [kd=0 -> slice jd-1, pd=1 classes | kd=1 -> slice jd, pd=0 | kd=2 ->
//     slice jd, pd=1] with zero weight rows for unreachable classes.
//   MODE_P5: the 5x5 stride-2 Conv2d layers of FeatureNet (conv1.0, conv2.0) as a planar
//     convolution over the (views, H, W) volume: the same even/odd planes (10 columns, 35 rows:
//     iw = 2*ow0-2+2j for kw = 0,2,4 at j, j+1, j+2; iw = 2*ow0-1+2j for kw = 1,3), 25 taps of
//     K = Cin, N = Cout, one output image per input image.
// How the input gets to shared memory and how the CTAs are scheduled:
//   * one TMA tiled load per (plane, 4 input channels) of a slice; out-of-bounds elements are
//     zero-filled by the TMA unit (= the zero padding);
//   * a plane is voxel-major [rows][9 or 10 columns][4 channels] (16 bytes per voxel, no
//     swizzle: 8 consecutive voxels are one wgmma core matrix), and every tap is a shifted view
//     of it (start address + rows*columns + column);
//   * MODE_S2 / MODE_P5: the even and odd input columns are two planes, each loaded by a TMA
//     whose box walks W with element stride 2 (tensor map elementStrides = {1,2,1,1,1});
//   * MODE_S2 with blocked input: one TMA load per channel quad brings the 33 rows of 18
//     input columns (2*w0-1 .. 2*w0+16) as one [33][18][4] run, 288 contiguous bytes per row,
//     into the space of the quad's two planes; the consumer warpgroups then rewrite it in place
//     into the even / odd planes (split_parities), so the GEMM reads the same planes as above;
//   * persistent CTAs, 9 warps (two consumer warpgroups of 64 GEMM rows each, one TMA
//     producer); the consumer keeps the accumulators of the output slices an input slice
//     reaches in registers and runs the epilogue of a slice as soon as it is complete.
//
// Replaces (reference):
//   ConvBnReLU(k=5, stride=2, pad=2)               models/modules.py:8-18, mvsnet.py:16,20
//   ConvBnReLU3D(stride=2)                         models/modules.py:21-31, mvsnet.py:65,68,71
//   ConvTranspose3d(k3,s2,p1,op1) + norm_act + skip models/mvsnet.py:74-87,99-101
#include "common.cuh"
#include "tc_common.cuh"
#include "tma_common.cuh"

namespace casmvs {
namespace tma2 {

using namespace casmvs::tc;
using namespace casmvs::tma;

enum { MODE_S2 = 0, MODE_T = 1, MODE_P5 = 2 };

struct Params {
  const float* bimg;   // pre-built B operand image [chunk][tap][CIN/4][BROWS][4] (tf32-rounded)
  const float* scale;  // [Cout]
  const float* shift;  // [Cout]
  const float* skip;   // output-shaped or null
  float* y;            // (B,Do,Ho,Wo,Cout)
  float slope;
  int B, Di, Hi, Wi, Do, Ho, Wo, Cout;     // Cout = channel count of the output tensor;
                                           // a CTA handles the COUT-channel chunk blockIdx.y
  tma::Work work;       // tiles over the M space (output for S2 and P5, input for T)
  int round_out;
  int x_blocked;       // x stored blocked by channel quads (tma::input_map); else channels-last
  int y_blocked;       // y and skip stored blocked by channel quads; else channels-last
};

template <int MODE, int CIN, int COUT>
struct Cfg {
  static constexpr int CQ = CIN / 4;
  static constexpr int BR = MODE == MODE_S2 ? 33 : MODE == MODE_T ? 17 : 35;   // brick rows
  static constexpr int BW = MODE == MODE_P5 ? 10 : 9;       // brick columns per plane
  static constexpr int PAR = MODE == MODE_T ? 1 : 2;        // column-parity planes
  static constexpr int NPL = PAR * CQ;                      // planes (= TMA loads) per slice
  static constexpr int kPlaneData = BR * BW * 16;
  static constexpr int kPlaneBytes = (kPlaneData + 127) / 128 * 128;
  static constexpr int kSlotBytes = NPL * kPlaneBytes;
  // MODE_S2, blocked input: the run of one channel quad, [BR][2 BW][4], at the quad's planes
  static constexpr int kRunData = BR * 2 * BW * 16;
  static_assert(MODE != MODE_S2 || kRunData == PAR * kPlaneData, "a run fills the quad's planes");
  // accumulator group (columns per output group) and B image rows per tap
  static constexpr int GW = MODE == MODE_T ? 8 * COUT : (COUT <= 16 ? 16 : 32);
  static constexpr int BROWS = MODE == MODE_S2 ? 3 * GW : MODE == MODE_T ? 12 * COUT : GW;
  static constexpr int NTAP = MODE == MODE_S2 ? 9 : MODE == MODE_T ? 4 : 25;   // A views per slice
  static constexpr int kWBytes = NTAP * CIN * BROWS * 4;
  static constexpr int kFixed = kWBytes + 2 * 32 * 4 + 192 + 1024;
  static constexpr int SLOTS = (kFixed + 4 * kSlotBytes <= 227 * 1024) ? 4
                               : (kFixed + 3 * kSlotBytes <= 227 * 1024) ? 3 : 2;
  static constexpr int kRingOff = 0;
  static constexpr int kWOff = SLOTS * kSlotBytes;
  static constexpr int kParamOff = kWOff + kWBytes;         // scale/shift [2][COUT pad 32]
  static constexpr int kBarOff = kParamOff + 2 * 32 * 4;
  // barriers: full[8] @0, empty[8] @64, weight image @128
  static constexpr int kTotal = kBarOff + 192 + 1024;
};

template <int MODE, int CIN, int COUT>
__global__ void __launch_bounds__(kConvThreads, 1)
conv3d_tma2_kernel(const __grid_constant__ CUtensorMap xmap, const Params p) {
  using C = Cfg<MODE, CIN, COUT>;
  constexpr int BW = C::BW, GW = C::GW, BROWS = C::BROWS;
  constexpr int SLOTS = C::SLOTS;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem;
  const uint32_t s_base = smem_align_1024(smem_raw, &smem);
  const uint32_t s_ring = s_base + C::kRingOff, s_w = s_base + C::kWOff,
                 s_bar = s_base + C::kBarOff;
  float* s_param = reinterpret_cast<float*>(smem + C::kParamOff);
  const Ring<SLOTS> ring{s_bar, s_bar + 64};
  const uint32_t bar_w = s_bar + 128;
  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int total_items = p.B * p.work.nchunks * p.work.tiles_h * p.work.tiles_w;
  const int Dm = MODE == MODE_T ? p.Di : p.Do;               // M-space depth

  // ---- one-time setup ----
  {
    const int t = threadIdx.x;
    ring.init(t, 1, kConsumerThreads);
    if (t == 2 * SLOTS) mbar_init(bar_w, 1);
    if (t <= 2 * SLOTS) fence_barrier_init();
  }
  const int co_base = blockIdx.y * COUT;
  stage_scale_shift<32>(s_param, p.scale, p.shift, co_base, COUT);
  end_prologue(ImageCopy{s_w, p.bimg + (size_t)blockIdx.y * (C::kWBytes / 4), C::kWBytes, bar_w});
  bool w_ready = false;                             // consumers: weight image has landed
  uint32_t gs = 0;                                  // slices processed before this item
  for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
    // work item: (b, chunk of groups along depth, M-space origin of the tile)
    const Item t = decode_item(item, p.work);
    const int b = t.b, h0 = t.h0, w0 = t.w0;
    const int g0 = t.chunk * p.work.dchunk, g1 = min(Dm, g0 + p.work.dchunk);
    const int ng = g1 - g0;                                  // output groups of this item
    // input slices walked: S2: s = 2*g0-1 .. 2*g1-1  (2*ng+1);  T: s = g0 .. g1  (ng+1)
    // P5: s = g0 .. g1-1 (every image is its own group)
    const int nslices = MODE == MODE_S2 ? 2 * ng + 1 : MODE == MODE_T ? ng + 1 : ng;
    const int s_first = MODE == MODE_S2 ? 2 * g0 - 1 : g0;

    if (warp == kProdWarp) {
      // ===================== producer: NPL TMA loads per slice =====================
      if (lane == 0) {
        for (int it = 0; it < nslices; ++it) {
          const uint32_t g = gs + it;
          const uint32_t dst = s_ring + ring.acquire(g) * C::kSlotBytes, full = ring.full_bar(g);
          mbar_expect_tx(full, C::NPL * C::kPlaneData);
          if (MODE == MODE_S2 && p.x_blocked) {
            // one contiguous run per channel quad, split into its planes by the consumers
#pragma unroll
            for (int q = 0; q < C::CQ; ++q) {
              const tma::Coords5 k =
                  tma::brick_coords(true, q, 2 * w0 - 1, 2 * h0 - 1, s_first + it, b);
              tma_load_5d(dst + q * C::PAR * C::kPlaneBytes, &xmap, full, k.c[0], k.c[1], k.c[2],
                          k.c[3], k.c[4]);
            }
          } else {
#pragma unroll
            for (int pl = 0; pl < C::NPL; ++pl) {
              // plane pl = PAR * (channel quad) + column parity
              const int q = pl / C::PAR, par = pl % C::PAR;
              const int wc = MODE == MODE_S2 ? 2 * w0 - 1 + par
                             : MODE == MODE_T ? w0 : 2 * w0 - 2 + par;
              const int hc = MODE == MODE_S2 ? 2 * h0 - 1 : MODE == MODE_T ? h0 : 2 * h0 - 2;
              const tma::Coords5 k = tma::brick_coords(MODE == MODE_T && p.x_blocked, q, wc, hc,
                                                       s_first + it, b);
              tma_load_5d(dst + pl * C::kPlaneBytes, &xmap, full, k.c[0], k.c[1], k.c[2], k.c[3],
                          k.c[4]);
            }
          }
        }
      }
      __syncwarp();
    } else {
      // ============ consumer warpgroups: wgmma into registers, then the epilogue ============
      const int wg = warp >> 2, wl = warp & 3;
      const int row0 = 64 * wg;
      constexpr uint32_t a_lbo = C::PAR * C::kPlaneBytes;     // next channel quad, same parity
      constexpr uint32_t a_sbo = (MODE == MODE_T ? 1 : 2) * BW * 16;
      constexpr uint32_t b_lbo = BROWS * 16, b_sbo = 128;
      const uint64_t a_desc0 = make_desc(s_ring + 8 * wg * a_sbo, a_lbo, a_sbo);
      const uint64_t b_desc0 = make_desc(s_w, b_lbo, b_sbo);
      // accumulators: S2 [group a-1 | group a] (2*GW columns), P5 [image] (GW), T [kd=0 block
      // of group it-1 | kd=1 block of group it | kd=2 block of group it] (12*COUT) plus the
      // pd=0 half of the previous group (4*COUT)
      constexpr int NACC = MODE == MODE_S2 ? 2 * GW : MODE == MODE_T ? 12 * COUT : GW;
      float acc[NACC / 2];
      float prev0[MODE == MODE_T ? 2 * COUT : 1];
#pragma unroll
      for (int i = 0; i < NACC / 2; ++i) acc[i] = 0.f;

      // issue all taps of one input slice: N columns from B row `row0b`
      auto issue = [&](auto n_tag, uint64_t a_s, int row0b) {
        constexpr int N = decltype(n_tag)::value;
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < C::NTAP; ++tap) {
          int a_tap, pl0;                            // voxel offset in a plane, column parity
          if (MODE == MODE_S2) {
            const int kh = tap / 3, kw = tap % 3;
            a_tap = kh * BW + (kw == 2 ? 1 : 0);
            pl0 = kw == 1 ? 1 : 0;
          } else if (MODE == MODE_P5) {
            const int kh = tap / 5, kw = tap % 5;
            a_tap = kh * BW + (kw >> 1);
            pl0 = kw & 1;
          } else {
            const int sh = tap >> 1, sw = tap & 1;
            a_tap = sh * BW + sw;
            pl0 = 0;
          }
#pragma unroll
          for (int k8 = 0; k8 < CIN / 8; ++k8) {
            const uint32_t a_off = ((2 * k8 * C::PAR + pl0) * C::kPlaneBytes + a_tap * 16) >> 4;
            const uint32_t b_off = (tap * (CIN * BROWS * 4) + k8 * 2 * BROWS * 16 + row0b * 16) >> 4;
            wgmma_tf32<N>(acc, a_s + a_off, b_desc0 + b_off);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
      };

      // MODE_S2, blocked input: the slot holds each channel quad as one [BR][2 BW][4] run
      // (input columns 2*w0-1 .. 2*w0+16 side by side) where its two planes go.  Column c of
      // the run belongs to plane c & 1, column c >> 1.  The planes of a quad overlap its run
      // and nothing else, so the quads are split in batches of up to four: every consumer thread
      // loads its voxels of the batch into registers, and stores them once all 256 have loaded.
      // A thread handles the same run voxels i = t + 256 k in every quad.  The stores are
      // generic-proxy writes that the wgmma (async proxy) read: each thread fences them before
      // the last barrier.
      constexpr int kRun = C::BR * 2 * BW;                           // voxels of one run
      constexpr int kPer = (kRun + kConsumerThreads - 1) / kConsumerThreads;
      constexpr int kBatch = C::CQ < 4 ? C::CQ : 4;                  // quads per batch
      static_assert(C::CQ % kBatch == 0, "whole batches");
      uint32_t run_off[kPer], plane_off[kPer];
#pragma unroll
      for (int k = 0; k < kPer; ++k) {
        const int i = threadIdx.x + k * kConsumerThreads;
        const int r = i / (2 * BW), c = i - r * (2 * BW);
        run_off[k] = i < kRun ? i * 16 : ~0u;                        // ~0u: no voxel
        plane_off[k] = (c & 1) * C::kPlaneBytes + (r * BW + (c >> 1)) * 16;
      }
      auto split_parities = [&](int slot) {
        unsigned char* s = smem + C::kRingOff + slot * C::kSlotBytes;
#pragma unroll
        for (int q0 = 0; q0 < C::CQ; q0 += kBatch) {
          float4 v[kBatch][kPer];
#pragma unroll
          for (int j = 0; j < kBatch; ++j)
#pragma unroll
            for (int k = 0; k < kPer; ++k)
              if (run_off[k] != ~0u)
                v[j][k] = *reinterpret_cast<const float4*>(
                    s + (q0 + j) * C::PAR * C::kPlaneBytes + run_off[k]);
          asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
#pragma unroll
          for (int j = 0; j < kBatch; ++j)
#pragma unroll
            for (int k = 0; k < kPer; ++k)
              if (run_off[k] != ~0u)
                *reinterpret_cast<float4*>(s + (q0 + j) * C::PAR * C::kPlaneBytes +
                                           plane_off[k]) = v[j][k];
        }
        fence_proxy_async();
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
      };

      // stores two adjacent channels (c, c+1) of output voxel (od, oh, ow)
      auto store2 = [&](int od, int oh, int ow, int c, float a0, float a1, bool has_skip) {
        const size_t o =
            tma::vol_offset(MODE != MODE_P5 && p.y_blocked, b, od, oh, ow, co_base + c, p.Do, p.Ho,
                            p.Wo, p.Cout);
        float v0 = fmaf(a0, s_param[c], s_param[32 + c]);
        float v1 = fmaf(a1, s_param[c + 1], s_param[32 + c + 1]);
        v0 = v0 >= 0.f ? v0 : v0 * p.slope;
        v1 = v1 >= 0.f ? v1 : v1 * p.slope;
        if (has_skip) {
          const float2 s2 = __ldg(reinterpret_cast<const float2*>(p.skip + o));
          v0 += s2.x; v1 += s2.y;
        }
        if (p.round_out) { v0 = to_tf32(v0); v1 = to_tf32(v1); }
        *reinterpret_cast<float2*>(p.y + o) = make_float2(v0, v1);
      };
      // The stores below read copies of the completed accumulator columns, never the
      // accumulators themselves: an accumulator register touched on a divergent path makes ptxas
      // serialize the wgmma of the next slice.
      // S2 / P5: output slice `od` from the GW columns in `src`
      auto store_plain = [&](const float* src, int od) {
        for_each_pair<0, GW>(src, wl, lane, [&](int r, int c, float a0, float a1) {
          const int m = row0 + r;
          const int mh = h0 + (m >> 3), mw = w0 + (m & 7);
          if (c < COUT && mh < p.Ho && mw < p.Wo) store2(od, mh, mw, c, a0, a1, false);
        });
      };
      // T, blocked output, COUT >= 16: the output voxels 2mw and 2mw+1 of one row come from the
      // parity classes (ph, 0) and (ph, 1), which this thread holds for the same channel pair
      // (c, c+1) (class columns cls*COUT + c).  Lanes l and l^1 hold the pairs c and c^2 of one
      // channel quad: they swap one class each, so that the even lane stores the whole quad of
      // voxel 2mw and the odd lane that of 2mw+1 -- one 32-byte sector per lane pair, not two
      // halves in different instructions.  Measured on conv9 (COUT = 16) this is 15-20 % faster
      // than the per-pair stores; on conv11 (COUT = 8) it is 20 % slower, so COUT = 8 (conv11,
      // conv7's 8-channel chunks) keeps the per-pair stores of store2.
      auto store_t_blocked = [&](const float* src, int od) {
        const bool odd = lane & 1;
        // element (quad cq of this CTA's chunk, output voxel (od, oh, ow)) at
        // yoff + cq * qstr + (oh * Wo + ow) * 4: 64-bit arithmetic once per slice
        const size_t qstr = (size_t)p.Do * p.Ho * p.Wo * 4;
        const size_t yoff = ((size_t)b * (p.Cout / 4) + co_base / 4) * qstr +
                            (size_t)od * p.Ho * p.Wo * 4;
#pragma unroll
        for (int ph = 0; ph < 2; ++ph) {
#pragma unroll
          for (int jj = 0; jj < COUT / 8; ++jj) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i0 = 4 * (2 * ph * (COUT / 8) + jj) + 2 * h;   // class (ph, 0)
              const int i1 = i0 + COUT / 2;                             // class (ph, 1)
              const int c = 8 * jj + 2 * (lane & 3);
              float e[4] = {src[i0], src[i0 + 1], src[i1], src[i1 + 1]};
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const float v = fmaf(e[k], s_param[c + (k & 1)], s_param[32 + c + (k & 1)]);
                e[k] = v >= 0.f ? v : v * p.slope;
              }
              const float s0 = __shfl_xor_sync(0xffffffffu, odd ? e[0] : e[2], 1);
              const float s1 = __shfl_xor_sync(0xffffffffu, odd ? e[1] : e[3], 1);
              float4 v = odd ? make_float4(s0, s1, e[2], e[3]) : make_float4(e[0], e[1], s0, s1);
              const int m = row0 + 16 * wl + (lane >> 2) + 8 * h;
              const int mh = h0 + (m >> 3), mw = w0 + (m & 7);
              if (mh >= p.Hi || mw >= p.Wi) continue;
              const size_t o = yoff + (c >> 2) * qstr +
                               (uint32_t)(((2 * mh + ph) * p.Wo + 2 * mw + (odd ? 1 : 0)) * 4);
              if (p.skip) {
                const float4 s4 = __ldg(reinterpret_cast<const float4*>(p.skip + o));
                v.x += s4.x; v.y += s4.y; v.z += s4.z; v.w += s4.w;
              }
              if (p.round_out) {
                v.x = to_tf32(v.x); v.y = to_tf32(v.y); v.z = to_tf32(v.z); v.w = to_tf32(v.w);
              }
              *reinterpret_cast<float4*>(p.y + o) = v;
            }
          }
        }
      };
      // T: input-slice group jd: pd=0 classes from prev0, pd=1 classes from `pd1` (acc block 0)
      auto store_t = [&](const float* pd1, int jd) {
        if (COUT >= 16 && p.y_blocked) {
          store_t_blocked(prev0, 2 * jd);
          store_t_blocked(pd1, 2 * jd + 1);
          return;
        }
        auto one = [&](int pd, int r, int col, float a0, float a1) {
          const int m = row0 + r;
          const int mh = h0 + (m >> 3), mw = w0 + (m & 7);
          if (mh >= p.Hi || mw >= p.Wi) return;
          const int cls = col / COUT, c = col % COUT;         // class (ph, pw) of this block
          const int ph = cls >> 1, pw = cls & 1;
          store2(2 * jd + pd, 2 * mh + ph, 2 * mw + pw, c, a0, a1, p.skip != nullptr);
        };
        for_each_pair<0, 4 * COUT>(prev0, wl, lane,
                                   [&](int r, int col, float a0, float a1) { one(0, r, col, a0, a1); });
        for_each_pair<0, 4 * COUT>(pd1, wl, lane,
                                   [&](int r, int col, float a0, float a1) { one(1, r, col, a0, a1); });
      };

      for (int it = 0; it < nslices; ++it) {
        const uint32_t g = gs + it;
        const int slot = ring.wait(g);
        if (!w_ready) { mbar_wait(bar_w, 0); w_ready = true; }
        const uint64_t a_s = a_desc0 + ((slot * C::kSlotBytes) >> 4);
        if constexpr (MODE == MODE_S2) {
          if (p.x_blocked) split_parities(slot);
          // B rows [W(kd=1) | W(kd=2) | W(kd=0)]
          if ((it & 1) == 0) issue(std::integral_constant<int, 2 * GW>{}, a_s, GW);  // kd=2 -> a-1, kd=0 -> a
          else issue(std::integral_constant<int, GW>{}, a_s, 0);                    // kd=1 -> a
        } else if constexpr (MODE == MODE_P5) {
#pragma unroll
          for (int i = 0; i < GW / 2; ++i) acc[i] = 0.f;
          issue(std::integral_constant<int, GW>{}, a_s, 0);
        } else {
          issue(std::integral_constant<int, 12 * COUT>{}, a_s, 0);
        }
        ring.release(g);                            // this thread's reads of the slot are done
        if constexpr (MODE == MODE_S2) {
          if ((it & 1) == 0) {
            // even walk index it = 2a: group a-1 is complete (its kd = 2 slice was this one)
            const int a = it >> 1;
            float done[GW / 2];
#pragma unroll
            for (int i = 0; i < GW / 2; ++i) {
              done[i] = acc[i];
              acc[i] = acc[GW / 2 + i];
              acc[GW / 2 + i] = 0.f;
            }
            if (a >= 1) store_plain(done, g0 + a - 1);
          }
        } else if constexpr (MODE == MODE_P5) {
          float done[GW / 2];
#pragma unroll
          for (int i = 0; i < GW / 2; ++i) done[i] = acc[i];
          store_plain(done, g0 + it);
        } else {
          float pd1[2 * COUT];
#pragma unroll
          for (int i = 0; i < 2 * COUT; ++i) pd1[i] = acc[i];
          if (it >= 1) store_t(pd1, g0 + it - 1);
          // roll: kd=1 block -> pd=0 half of the previous group, kd=2 block -> block 0
#pragma unroll
          for (int i = 0; i < 2 * COUT; ++i) {
            prev0[i] = acc[2 * COUT + i];
            acc[i] = acc[4 * COUT + i];
            acc[2 * COUT + i] = 0.f;
            acc[4 * COUT + i] = 0.f;
          }
        }
      }
    }
    gs += nslices;
  }
}

// B operand image [chunk][tap][cq][row][4], tf32-rounded
template <int MODE, int CIN, int COUT>
__global__ void build_image_tma2_kernel(const float* __restrict__ wpk, float* __restrict__ img,
                                        int cout_total) {
  using C = Cfg<MODE, CIN, COUT>;
  constexpr int CQ = C::CQ, GW = C::GW, BROWS = C::BROWS;
  constexpr int per = C::NTAP * CIN * BROWS;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < per * (cout_total / COUT);
       t += gridDim.x * blockDim.x) {
    const int ck = t / per, i = t - ck * per;
    const int jq = i & 3;
    const int row = (i >> 2) % BROWS;
    const int r = (i >> 2) / BROWS;          // tap*CQ + cq
    const int cq = r % CQ, tap = r / CQ;
    const int ci = cq * 4 + jq;
    int kd = -1, kh = -1, kw = -1, co = -1;
    if (MODE == MODE_S2) {
      // rows [W(kd=1) | W(kd=2) | W(kd=0)], tap = kh*3+kw
      const int g = row / GW;
      co = row % GW;
      kd = g == 0 ? 1 : g == 1 ? 2 : 0;
      kh = tap / 3; kw = tap % 3;
      if (co >= COUT) kd = -1;
    } else {
      // tap = sh*2+sw; rows: block 0 kd=0 (pd=1), block 1 kd=1 (pd=0), block 2 kd=2 (pd=1);
      // inside a block: class (ph,pw) = 2*ph+pw, then co
      const int sh = tap >> 1, sw = tap & 1;
      const int blk = row / (4 * COUT);
      const int cls = (row / COUT) & 3;
      co = row % COUT;
      const int ph = cls >> 1, pw = cls & 1;
      kd = blk;
      kh = sh == 0 ? (ph == 0 ? 1 : 2) : (ph == 1 ? 0 : -1);
      kw = sw == 0 ? (pw == 0 ? 1 : 2) : (pw == 1 ? 0 : -1);
      if (kh < 0 || kw < 0) kd = -1;
    }
    float v = 0.f;
    if (kd >= 0)
      v = to_tf32(__ldg(wpk + ((size_t)((kd * 3 + kh) * 3 + kw) * CIN + ci) * cout_total +
                        ck * COUT + co));
    img[t] = v;
  }
}

// MODE_P5 image [tap = kh*5+kw][cq][co (GW rows)][4] from the torch Conv2d weight (Cout,Cin,5,5)
template <int CIN, int COUT>
__global__ void build_image_p5_kernel(const float* __restrict__ wt, float* __restrict__ img) {
  using C = Cfg<MODE_P5, CIN, COUT>;
  constexpr int CQ = C::CQ, GW = C::GW;
  constexpr int total = 25 * CIN * GW;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    const int jq = t & 3;
    const int co = (t >> 2) % GW;
    const int r = (t >> 2) / GW;             // tap*CQ + cq
    const int cq = r % CQ, tap = r / CQ;
    const int ci = cq * 4 + jq;
    img[t] = co < COUT ? to_tf32(__ldg(wt + ((size_t)co * CIN + ci) * 25 + tap)) : 0.f;
  }
}

// The B operand image of a layer (all its COUT-channel chunks).
template <int MODE, int CIN, int COUT>
static int tma2_image(const float* wpk, int cout_total, cudaStream_t st, ImageRef* ir) {
  using C = Cfg<MODE, CIN, COUT>;
  return cached_image(wpk, 2000 + MODE * 10000 + CIN * 100 + COUT,
                      (size_t)C::kWBytes * (cout_total / COUT), st, ir, "conv3d_tma2/build_image",
                      [&](float* img) {
                        if constexpr (MODE == MODE_P5)
                          build_image_p5_kernel<CIN, COUT><<<32, 256, 0, st>>>(wpk, img);
                        else
                          build_image_tma2_kernel<MODE, CIN, COUT><<<64, 256, 0, st>>>(wpk, img,
                                                                                       cout_total);
                      });
}

// MODE_S2 / MODE_P5: output = (in - 1) / 2 + 1 along H and W (and D for MODE_S2); MODE_T:
// output = 2x input.  A CTA computes a COUT-channel slice of a.Cout.
template <int MODE, int CIN, int COUT>
static int launch2(const ConvArgs& a, cudaStream_t st) {
  using C = Cfg<MODE, CIN, COUT>;
  static_assert(C::kTotal <= 227 * 1024, "shared memory budget");
  auto kfn = conv3d_tma2_kernel<MODE, CIN, COUT>;
  static std::atomic<bool> attr_set[kMaxDevices];
  if (int rc = opt_in_smem(kfn, C::kTotal, attr_set, "conv3d_tma2")) return rc;
  Params p;
  p.scale = a.scale; p.shift = a.shift; p.skip = a.skip; p.y = a.y;
  p.slope = a.slope; p.B = a.B; p.Di = a.D; p.Hi = a.h; p.Wi = a.w; p.Cout = a.Cout;
  p.Do = MODE == MODE_T ? 2 * a.D : MODE == MODE_S2 ? (a.D - 1) / 2 + 1 : a.D;
  p.Ho = MODE == MODE_T ? 2 * a.h : (a.h - 1) / 2 + 1;
  p.Wo = MODE == MODE_T ? 2 * a.w : (a.w - 1) / 2 + 1;
  p.round_out = a.round_out;
  p.x_blocked = (a.layout & kLayoutXBlocked) ? 1 : 0;
  p.y_blocked = (a.layout & kLayoutYBlocked) ? 1 : 0;
  // S2: box {4, 17 traversed -> 9 loaded, 33, 1, 1} walking W with stride 2, or, blocked, one
  // run of 18 voxels x 33 rows {72, 33, 1, 1, 1}; T: {4, 9, 17}
  // P5: box {4, 19 traversed -> 10 loaded, 35, 1, 1} walking W with stride 2
  CUtensorMap map;
  const int rc =
      MODE == MODE_S2   ? (p.x_blocked ? tma::input_map(&map, a.x, p.B, p.Di, p.Hi, p.Wi, CIN,
                                                        2 * C::BW, C::BR, 1, true)
                                       : tma::input_map(&map, a.x, p.B, p.Di, p.Hi, p.Wi, CIN, 17,
                                                        C::BR, 2))
      : MODE == MODE_P5 ? tma::input_map(&map, a.x, p.B, p.Di, p.Hi, p.Wi, CIN, 19, C::BR, 2)
                        : tma::input_map(&map, a.x, p.B, p.Di, p.Hi, p.Wi, CIN, C::BW, C::BR, 1,
                                         p.x_blocked);
  if (rc) return rc;
  const int Dm = MODE == MODE_T ? p.Di : p.Do;
  const int Hm = MODE == MODE_T ? p.Hi : p.Ho, Wm = MODE == MODE_T ? p.Wi : p.Wo;
  p.work.tiles_w = (Wm + kTileW - 1) / kTileW;
  p.work.tiles_h = (Hm + kTileH - 1) / kTileH;
  const int nco = p.Cout / COUT;
  const tma::Sizing z = tma::size_persistent(
      kfn, C::kTotal, nco, (long)p.B * p.work.tiles_w * p.work.tiles_h, Dm, 32,
      MODE == MODE_S2 ? 2 : 1, MODE == MODE_S2 ? 1 : MODE == MODE_T ? 1 : 0);
  p.work.dchunk = z.dchunk;
  p.work.nchunks = z.nchunks;
  ImageRef ir;
  if (int rc = tma2_image<MODE, CIN, COUT>(a.wpk, p.Cout, st, &ir)) return rc;
  p.bimg = ir.img;
  tma::launch_pdl(ir.settled, kfn, z.grid, kConvThreads, C::kTotal, st, map, p);
  return after_launch("conv3d_tma2");
}

// Coverage: the CostRegNet layer shapes this kernel is instantiated for (stride 2).  The
// stride-2 epilogue has no skip input.
struct Shape {
  int kind, cin, cout;
  bool skip;
  ConvLauncher run;
};
static const Shape kShapes[] = {
    {CASMVS_CONV, 8, 16, false, launch2<MODE_S2, 8, 16>},
    {CASMVS_CONV, 16, 32, false, launch2<MODE_S2, 16, 32>},
    {CASMVS_CONV, 32, 64, false, launch2<MODE_S2, 32, 16>},
    {CASMVS_CONV_TRANSPOSE, 16, 8, true, launch2<MODE_T, 16, 8>},
    {CASMVS_CONV_TRANSPOSE, 32, 16, true, launch2<MODE_T, 32, 16>},
    {CASMVS_CONV_TRANSPOSE, 64, 32, true, launch2<MODE_T, 64, 8>},
};

}  // namespace tma2

ConvLauncher conv3d_tma2_find(int Cin, int Cout, int kind, int stride, bool skip) {
  if (stride != 2) return nullptr;
  for (const tma2::Shape& s : tma2::kShapes)
    if (s.kind == kind && s.cin == Cin && s.cout == Cout && (s.skip || !skip)) return s.run;
  return nullptr;
}

int conv3d_tma2_conv11_image(const float* wpk, cudaStream_t st, tc::ImageRef* ir) {
  return tma2::tma2_image<tma2::MODE_T, 16, 8>(wpk, 8, st, ir);
}

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_conv2d_5x5s2_fwd(const float* x, const float* w, const float* shift,
                                       float slope, float* y, int N, int Cin, int Cout, int H,
                                       int W, int round_tf32, void* stream) {
  CASMVS_REQUIRE_ALIGNED("conv2d_5x5s2", x, 16);
  CASMVS_REQUIRE(x && w && y, "conv2d_5x5s2: null pointer");
  CASMVS_REQUIRE(N >= 0 && H >= 2 && W >= 2, "conv2d_5x5s2: bad dims");
  if (N == 0) return 0;
  const ConvArgs a{x, w, nullptr, shift, nullptr, y, slope, 1, Cin, Cout, N, H, W, 0,
                   round_tf32 ? 1 : 0};
  cudaStream_t st = as_stream(stream);
  if (Cin == 8 && Cout == 16) return tma2::launch2<tma2::MODE_P5, 8, 16>(a, st);
  if (Cin == 16 && Cout == 32) return tma2::launch2<tma2::MODE_P5, 16, 32>(a, st);
  set_error("conv2d_5x5s2: only the FeatureNet shapes 8->16 and 16->32 are built (got %d->%d)",
            Cin, Cout);
  return -1;
}
