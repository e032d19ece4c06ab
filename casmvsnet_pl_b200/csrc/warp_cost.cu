// K1 — fused homography plane-sweep warp + bilinear sample + cost reduction.
//
// Replaces (reference, paths relative to /root/reference):
//   homo_warp                      models/modules.py:52-92   (called V-1 times)
//   variance accumulation          models/mvsnet.py:137-141,147-156,166-168
//   group-wise correlation         models/mvsnet.py:143-144,158-162,170-172
// The (B,V-1,C,D,h,w) warped volumes never exist in HBM: every thread owns one
// reference pixel x 8 channels, walks the D depth planes, gathers the 4 bilinear
// taps of every source view straight from the channels-last feature maps
// (a tap = 32 contiguous bytes per thread, 32*C/8 per pixel) and keeps the
// running sum / sum of squares in registers.
//
// HBM model (DESIGN.md): read V*C*h*w feature floats once (they live in L2 for
// the whole launch), read D*h*w hypotheses once, write Cout*D*h*w cost floats
// once.  The kernel is write-bound.
#include "k1_common.cuh"

namespace casmvs {

constexpr int kMaxSrc = 15;      // V-1 supported by the smem projection table
constexpr int kK1Threads = 128;

struct Taps {
  int o00, o01, o10, o11;  // float offsets of the 4 taps (channel 0) inside the view
  float w00, w01, w10, w11;
  bool any;
};

// Sample position for one source view; follows models/modules.py:72-84 +
// ATen grid_sampler_2d (bilinear, zeros padding, align_corners=True).
__device__ __forceinline__ Taps make_taps(float qx, float qy, float qz, int h, int w, int C) {
  Taps t;
  t.any = false;
  t.o00 = t.o01 = t.o10 = t.o11 = 0;
  t.w00 = t.w01 = t.w10 = t.w11 = 0.f;
  // q_z <= 1e-7 is sent to (w,h): fully outside => zeros (modules.py:76-79)
  if (!(qz > 1e-7f)) return t;
  float rz = __frcp_rn(qz);
  float u = qx * rz, v = qy * rz;
  // bounds are tested in float BEFORE any int conversion (|u| may be huge / NaN)
  if (!(u > -1.f && u < (float)w && v > -1.f && v < (float)h)) return t;
  float x0f = floorf(u), y0f = floorf(v);
  int x0 = (int)x0f, y0 = (int)y0f;
  float wx1 = u - x0f, wx0 = (x0f + 1.f) - u;   // ATen: (ix_se - ix), (ix - ix_nw)
  float wy1 = v - y0f, wy0 = (y0f + 1.f) - v;
  int x1 = x0 + 1, y1 = y0 + 1;
  if (x0 < 0) { wx0 = 0.f; x0 = 0; }
  if (x1 > w - 1) { wx1 = 0.f; x1 = w - 1; }
  if (y0 < 0) { wy0 = 0.f; y0 = 0; }
  if (y1 > h - 1) { wy1 = 0.f; y1 = h - 1; }
  t.w00 = wx0 * wy0; t.w01 = wx1 * wy0; t.w10 = wx0 * wy1; t.w11 = wx1 * wy1;
  t.o00 = (y0 * w + x0) * C; t.o01 = (y0 * w + x1) * C;
  t.o10 = (y1 * w + x0) * C; t.o11 = (y1 * w + x1) * C;
  t.any = true;
  return t;
}

__device__ __forceinline__ void blend8(const float* __restrict__ base, const Taps& t,
                                       float (&r)[kCPT]) {
  // tap order nw, ne, sw, se like ATen
  float4 a0 = ldg4(base + t.o00), a1 = ldg4(base + t.o00 + 4);
  float4 b0 = ldg4(base + t.o01), b1 = ldg4(base + t.o01 + 4);
  float4 c0 = ldg4(base + t.o10), c1 = ldg4(base + t.o10 + 4);
  float4 d0 = ldg4(base + t.o11), d1 = ldg4(base + t.o11 + 4);
  r[0] = fmaf(d0.x, t.w11, fmaf(c0.x, t.w10, fmaf(b0.x, t.w01, a0.x * t.w00)));
  r[1] = fmaf(d0.y, t.w11, fmaf(c0.y, t.w10, fmaf(b0.y, t.w01, a0.y * t.w00)));
  r[2] = fmaf(d0.z, t.w11, fmaf(c0.z, t.w10, fmaf(b0.z, t.w01, a0.z * t.w00)));
  r[3] = fmaf(d0.w, t.w11, fmaf(c0.w, t.w10, fmaf(b0.w, t.w01, a0.w * t.w00)));
  r[4] = fmaf(d1.x, t.w11, fmaf(c1.x, t.w10, fmaf(b1.x, t.w01, a1.x * t.w00)));
  r[5] = fmaf(d1.y, t.w11, fmaf(c1.y, t.w10, fmaf(b1.y, t.w01, a1.y * t.w00)));
  r[6] = fmaf(d1.z, t.w11, fmaf(c1.z, t.w10, fmaf(b1.z, t.w01, a1.z * t.w00)));
  r[7] = fmaf(d1.w, t.w11, fmaf(c1.w, t.w10, fmaf(b1.w, t.w01, a1.w * t.w00)));
}

// NSRC > 0: number of source views known at compile time (per-view R*(x,y,1) stays
// in registers); NSRC == 0: generic run-time V.  CT: compile-time C (0 = generic).
// grid = (pixel-thread blocks, B, depth chunks of `dchunk` planes).  Needs h,w >= 2.
template <int NSRC, int CT, bool GWC, bool OUT_NHWC>
__global__ void __launch_bounds__(kK1Threads, 4)
warp_cost_kernel(const float* __restrict__ feats,   // (B,V,h,w,C)
                 const float* __restrict__ proj,    // (B,V-1,3,4)
                 const float* __restrict__ dv,      // (B,D,h,w)
                 float* __restrict__ cost, int V, int C_rt, int D, int h, int w, int G,
                 int dchunk, int round_tf32) {
  __shared__ float s_proj[kMaxSrc * 12];
  const int C = CT > 0 ? CT : C_rt;
  const int b = blockIdx.y;
  const int nsrc = NSRC > 0 ? NSRC : V - 1;
  for (int i = threadIdx.x; i < nsrc * 12; i += blockDim.x)
    s_proj[i] = proj[(size_t)b * nsrc * 12 + i];
  __syncthreads();

  const int tpp = C / kCPT;                       // threads per pixel
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int pix = gtid / tpp;
  const int sub = gtid - pix * tpp;
  const int c0 = sub * kCPT;
  const int hw = h * w;
  const bool active = pix < hw;
  const int pixc = active ? pix : hw - 1;         // inactive lanes still take part in shuffles
  const int y = pixc / w, x = pixc - y * w;
  const float xf = (float)x, yf = (float)y;
  const int row_floats = w * C;

  const size_t view_stride = (size_t)hw * C;
  const float* fb = feats + (size_t)b * V * view_stride + c0;

  const Tex8 ref = ldg256(fb + (size_t)pixc * C);
  u64 refsq[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) refsq[k] = mul2(ref.v[k], ref.v[k]);

  constexpr int NV = NSRC > 0 ? NSRC : 1;
  float ax[NV], ay[NV], az[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const float* P = s_proj + v * 12;
    ax[v] = fmaf(P[0], xf, fmaf(P[1], yf, P[2]));   // R*(x,y,1)   (modules.py:72)
    ay[v] = fmaf(P[4], xf, fmaf(P[5], yf, P[6]));
    az[v] = fmaf(P[8], xf, fmaf(P[9], yf, P[10]));
  }

  const float inv_v = 1.f / (float)V;
  const u64 inv_v2 = pk2(inv_v, inv_v), ninv_v2 = pk2(-inv_v, -inv_v);
  const int cpg = GWC ? C / G : 1;                // channels per group
  const int cout = GWC ? G : C;
  const float* dvp = dv + (size_t)b * D * hw + pixc;
  const int d_begin = blockIdx.z * dchunk;
  const int d_end = min(D, d_begin + dchunk);

  float tx[NV], ty[NV], tz[NV];                   // T of each view (modules.py:64)
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    tx[v] = s_proj[v * 12 + 3]; ty[v] = s_proj[v * 12 + 7]; tz[v] = s_proj[v * 12 + 11];
  }
  const float* dptr = dvp + (size_t)d_begin * hw;
  float depth_next = d_begin < d_end ? __ldg(dptr) : 1.f;

  for (int d = d_begin; d < d_end; ++d) {
    const float depth = depth_next;
    dptr += hw;
    if (d + 1 < d_end) depth_next = __ldg(dptr);  // prefetch: off the dependent chain
    const float inv_d = rcp_approx(depth);
    u64 S[4], Q[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      S[k] = GWC ? 0ull : ref.v[k];               // gwc: reference NOT in the sum (mvsnet.py:144)
      Q[k] = refsq[k];
    }
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      for (int vv = (NSRC > 0 ? v : 0); vv < (NSRC > 0 ? v + 1 : nsrc); ++vv) {
        float qx, qy, qz;
        if (NSRC > 0) {
          qx = fmaf(tx[v], inv_d, ax[v]);
          qy = fmaf(ty[v], inv_d, ay[v]);
          qz = fmaf(tz[v], inv_d, az[v]);
        } else {
          const float* P = s_proj + vv * 12;
          qx = fmaf(P[3], inv_d, fmaf(P[0], xf, fmaf(P[1], yf, P[2])));
          qy = fmaf(P[7], inv_d, fmaf(P[4], xf, fmaf(P[5], yf, P[6])));
          qz = fmaf(P[11], inv_d, fmaf(P[8], xf, fmaf(P[9], yf, P[10])));
        }
        gather_sample<CT>(fb + (size_t)(vv + 1) * view_stride, qx, qy, qz, h, w, C, row_floats,
                          [&](int k, u64 r) {
                            S[k] = add2(S[k], r);
                            if (!GWC) Q[k] = fma2(r, r, Q[k]);
                          });
      }
    }

    if (!GWC) {
      u64 o[4];
      variance(S, Q, inv_v2, ninv_v2, round_tf32, o);
      if (active) {
        if (OUT_NHWC) {
          stg256(cost + ((size_t)(b * D + d) * hw + pix) * C + c0, o);
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float lo, hi;
            unpk2(o[k], lo, hi);
            cost[((size_t)(b * C + c0 + 2 * k) * D + d) * hw + pix] = lo;
            cost[((size_t)(b * C + c0 + 2 * k + 1) * D + d) * hw + pix] = hi;
          }
        }
      }
    } else {
      // cost[g] = mean_{c in g}(S_c * ref_c) / (V-1)     (mvsnet.py:170-172)
      float p[kCPT];
#pragma unroll
      for (int k = 0; k < 4; ++k) unpk2(mul2(S[k], ref.v[k]), p[2 * k], p[2 * k + 1]);
      const float inv_cpg = 1.f / (float)cpg;
      const float vm1 = (float)(V - 1);
      if (cpg >= kCPT) {
        // one group spans cpg/8 neighbouring threads: reduce with shuffles
        float s = ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
        for (int off = 1; off < cpg / kCPT; off <<= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        const int g = c0 / cpg;
        if (active && (c0 % cpg) == 0) {
          float val = __fdiv_rn(s * inv_cpg, vm1);
          if (round_tf32) val = round_tf32_f(val);
          if (OUT_NHWC) cost[((size_t)(b * D + d) * hw + pix) * cout + g] = val;
          else cost[((size_t)(b * cout + g) * D + d) * hw + pix] = val;
        }
      } else {
        // cpg in {1,2,4}: this thread owns 8/cpg whole groups
        const int ng = kCPT / cpg;
        const int g0 = c0 / cpg;
        float o[kCPT];
#pragma unroll
        for (int k = 0; k < kCPT; ++k) o[k] = 0.f;
        if (cpg == 1) {
#pragma unroll
          for (int k = 0; k < kCPT; ++k) o[k] = p[k];
        } else if (cpg == 2) {
#pragma unroll
          for (int k = 0; k < 4; ++k) o[k] = p[2 * k] + p[2 * k + 1];
        } else {
#pragma unroll
          for (int k = 0; k < 2; ++k)
            o[k] = (p[4 * k] + p[4 * k + 1]) + (p[4 * k + 2] + p[4 * k + 3]);
        }
        if (active) {
#pragma unroll
          for (int k = 0; k < kCPT; ++k) {
            if (k < ng) {
              float val = __fdiv_rn(o[k] * inv_cpg, vm1);
              if (round_tf32) val = round_tf32_f(val);
              if (OUT_NHWC) cost[((size_t)(b * D + d) * hw + pix) * cout + g0 + k] = val;
              else cost[((size_t)(b * cout + g0 + k) * D + d) * hw + pix] = val;
            }
          }
        }
      }
    }
  }
}

// Stand-alone homo_warp: one thread = one pixel x 8 channels, all planes.
template <bool OUT_NHWC>
__global__ void __launch_bounds__(kK1Threads)
homo_warp_kernel(const float* __restrict__ src,   // (B,h,w,C)
                 const float* __restrict__ proj,  // (B,3,4)
                 const float* __restrict__ dv, float* __restrict__ out, int C, int D, int h,
                 int w) {
  const int b = blockIdx.y;
  const float* P = proj + (size_t)b * 12;
  const int tpp = C / kCPT;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int pix = gtid / tpp;
  const int c0 = (gtid - pix * tpp) * kCPT;
  const int hw = h * w;
  if (pix >= hw) return;
  const int y = pix / w, x = pix - y * w;
  const float xf = (float)x, yf = (float)y;
  const float ax = fmaf(P[0], xf, fmaf(P[1], yf, P[2]));
  const float ay = fmaf(P[4], xf, fmaf(P[5], yf, P[6]));
  const float az = fmaf(P[8], xf, fmaf(P[9], yf, P[10]));
  const float* sb = src + (size_t)b * hw * C + c0;
  for (int d = 0; d < D; ++d) {
    const float inv_d = __frcp_rn(__ldg(dv + ((size_t)b * D + d) * hw + pix));
    Taps t = make_taps(fmaf(P[3], inv_d, ax), fmaf(P[7], inv_d, ay), fmaf(P[11], inv_d, az),
                       h, w, C);
    float r[kCPT];
#pragma unroll
    for (int k = 0; k < kCPT; ++k) r[k] = 0.f;
    if (t.any) blend8(sb, t, r);
    if (OUT_NHWC) {
      float* op = out + ((size_t)(b * D + d) * hw + pix) * C + c0;
      st4(op, make_float4(r[0], r[1], r[2], r[3]));
      st4(op + 4, make_float4(r[4], r[5], r[6], r[7]));
    } else {
#pragma unroll
      for (int k = 0; k < kCPT; ++k) out[((size_t)(b * C + c0 + k) * D + d) * hw + pix] = r[k];
    }
  }
}

// (N,R,S) -> (N,S,R) through a 32x33 smem tile; tiles are flattened into grid.x.
__global__ void transpose_rs_kernel(const float* __restrict__ in, float* __restrict__ out,
                                    size_t R, size_t S, unsigned tiles_s) {
  __shared__ float tile[32][33];
  const size_t n = blockIdx.y;
  const float* ip = in + n * R * S;
  float* op = out + n * R * S;
  const size_t s0 = (size_t)(blockIdx.x % tiles_s) * 32;
  const size_t r0 = (size_t)(blockIdx.x / tiles_s) * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    size_t r = r0 + j, s = s0 + threadIdx.x;
    tile[j][threadIdx.x] = (r < R && s < S) ? ip[r * S + s] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    size_t s = s0 + j, r = r0 + threadIdx.x;
    if (r < R && s < S) op[s * R + r] = tile[threadIdx.x][j];
  }
}

static int launch_transpose(const float* in, float* out, int N, size_t R, size_t S,
                            cudaStream_t st, const char* what) {
  if (N == 0 || R == 0 || S == 0) return 0;
  dim3 blk(32, 8);
  size_t tiles_s = (S + 31) / 32, tiles_r = (R + 31) / 32;
  CASMVS_REQUIRE(tiles_s * tiles_r < (1ull << 31) && N <= 65535, "%s: dims too large", what);
  dim3 grd((unsigned)(tiles_s * tiles_r), (unsigned)N);
  transpose_rs_kernel<<<grd, blk, 0, st>>>(in, out, R, S, (unsigned)tiles_s);
  return after_launch(what);
}

template <int NSRC, int CT>
static void launch_k1(bool gwc, bool nhwc, dim3 grd, cudaStream_t st, const float* f,
                      const float* p, const float* dv, float* cost, int V, int C, int D, int h,
                      int w, int G, int dchunk, int rnd) {
  if (gwc) {
    if (nhwc) warp_cost_kernel<NSRC, CT, true, true><<<grd, kK1Threads, 0, st>>>(f, p, dv, cost, V, C, D, h, w, G, dchunk, rnd);
    else warp_cost_kernel<NSRC, CT, true, false><<<grd, kK1Threads, 0, st>>>(f, p, dv, cost, V, C, D, h, w, G, dchunk, rnd);
  } else {
    if (nhwc) warp_cost_kernel<NSRC, CT, false, true><<<grd, kK1Threads, 0, st>>>(f, p, dv, cost, V, C, D, h, w, G, dchunk, rnd);
    else warp_cost_kernel<NSRC, CT, false, false><<<grd, kK1Threads, 0, st>>>(f, p, dv, cost, V, C, D, h, w, G, dchunk, rnd);
  }
}

template <int NSRC>
static void launch_k1_c(bool gwc, bool nhwc, dim3 grd, cudaStream_t st, const float* f,
                        const float* p, const float* dv, float* cost, int V, int C, int D, int h,
                        int w, int G, int dchunk, int rnd) {
  switch (C) {
    case 8: launch_k1<NSRC, 8>(gwc, nhwc, grd, st, f, p, dv, cost, V, C, D, h, w, G, dchunk, rnd); break;
    case 16: launch_k1<NSRC, 16>(gwc, nhwc, grd, st, f, p, dv, cost, V, C, D, h, w, G, dchunk, rnd); break;
    case 32: launch_k1<NSRC, 32>(gwc, nhwc, grd, st, f, p, dv, cost, V, C, D, h, w, G, dchunk, rnd); break;
    default: launch_k1<NSRC, 0>(gwc, nhwc, grd, st, f, p, dv, cost, V, C, D, h, w, G, dchunk, rnd); break;
  }
}

}  // namespace casmvs

using namespace casmvs;

extern "C" size_t casmvs_warp_cost_workspace_bytes(int feat_layout, int B, int V, int C, int h,
                                                   int w) {
  if (feat_layout == CASMVS_NHWC) return 0;
  return (size_t)B * V * C * h * w * sizeof(float);
}

// Every K1 kernel reads the channels-last features (feats, or the workspace NCHW features are
// re-laid-out into) in 16-byte vectors, and writes a channels-last cost volume in vectors of up
// to 16 bytes.
extern "C" int casmvs_warp_cost_fwd(const float* feats, int feat_layout, const float* proj,
                                    const float* depth_values, float* cost, int cost_layout,
                                    int B, int V, int C, int D, int h, int w, int num_groups,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  if (feat_layout == CASMVS_NHWC) CASMVS_REQUIRE_ALIGNED("warp_cost", feats, 16);
  else CASMVS_REQUIRE_ALIGNED("warp_cost", workspace, 16);
  if ((cost_layout & ~CASMVS_ROUND_TF32) == CASMVS_NHWC) CASMVS_REQUIRE_ALIGNED("warp_cost", cost, 16);
  CASMVS_REQUIRE(feats && proj && depth_values && cost, "warp_cost: null pointer");
  CASMVS_REQUIRE(B >= 0 && V >= 2 && C > 0 && D > 0 && h >= 2 && w >= 2, "warp_cost: bad dims (h,w >= 2)");
  CASMVS_REQUIRE(V - 1 <= kMaxSrc, "warp_cost: at most %d source views", kMaxSrc);
  CASMVS_REQUIRE(C % kCPT == 0, "warp_cost: C must be a multiple of %d (got %d)", kCPT, C);
  CASMVS_REQUIRE(C / kCPT <= 32 && (32 % (C / kCPT)) == 0, "warp_cost: C/8 must divide 32");
  CASMVS_REQUIRE(num_groups >= 1 && C % num_groups == 0, "warp_cost: C %% num_groups != 0");
  const bool gwc = num_groups > 1;
  if (gwc) {
    int cpg = C / num_groups;
    CASMVS_REQUIRE((cpg & (cpg - 1)) == 0, "warp_cost: C/num_groups must be a power of two");
  }
  CASMVS_REQUIRE((size_t)h * w * C < (1u << 31), "warp_cost: view too large for 32-bit offsets");
  CASMVS_REQUIRE(B <= 65535, "warp_cost: B too large");
  if (B == 0) return 0;
  cudaStream_t st = as_stream(stream);
  const float* f = feats;
  if (feat_layout == CASMVS_NCHW) {
    size_t need = casmvs_warp_cost_workspace_bytes(feat_layout, B, V, C, h, w);
    CASMVS_REQUIRE(workspace && workspace_bytes >= need,
                   "warp_cost: workspace too small (%zu < %zu)", workspace_bytes, need);
    int rc = launch_transpose(feats, (float*)workspace, B * V, (size_t)C, (size_t)h * w, st,
                              "warp_cost/nchw_to_nhwc");
    if (rc) return rc;
    f = (const float*)workspace;
  } else {
    CASMVS_REQUIRE(feat_layout == CASMVS_NHWC, "warp_cost: bad feat_layout");
  }
  const int rnd = (cost_layout & CASMVS_ROUND_TF32) ? 1 : 0;
  cost_layout &= ~CASMVS_ROUND_TF32;
  CASMVS_REQUIRE(cost_layout == CASMVS_NCHW || cost_layout == CASMVS_NHWC,
                 "warp_cost: bad cost_layout");
  const bool nhwc = cost_layout == CASMVS_NHWC;
  const long threads = (long)h * w * (C / kCPT);
  const unsigned xblocks = (unsigned)((threads + kK1Threads - 1) / kK1Threads);
  if (StagedK1 run = nhwc ? warp_cost_staged(V, C, num_groups) : nullptr) {
    const Hyp hyp{depth_values, nullptr, nullptr, nullptr, 0.f, 0.f};
    return run(f, proj, hyp, cost, B, D, h, w, rnd, 0, kLadderUniform, st);
  }
  // depth chunks: enough CTAs to fill every SM several times over, but chunks long
  // enough (>= 8 planes) for the texel-window cache to pay off
  int dchunk = D;
  const long want_ctas = (long)num_sms() * 16;
  while (dchunk > 8 && (long)xblocks * B * ((D + dchunk - 1) / dchunk) < want_ctas)
    dchunk = (dchunk + 1) / 2;
  dim3 grd(xblocks, (unsigned)B, (unsigned)((D + dchunk - 1) / dchunk));
  switch (V - 1) {
    case 1: launch_k1_c<1>(gwc, nhwc, grd, st, f, proj, depth_values, cost, V, C, D, h, w, num_groups, dchunk, rnd); break;
    case 2: launch_k1_c<2>(gwc, nhwc, grd, st, f, proj, depth_values, cost, V, C, D, h, w, num_groups, dchunk, rnd); break;
    case 4: launch_k1_c<4>(gwc, nhwc, grd, st, f, proj, depth_values, cost, V, C, D, h, w, num_groups, dchunk, rnd); break;
    case 6: launch_k1_c<6>(gwc, nhwc, grd, st, f, proj, depth_values, cost, V, C, D, h, w, num_groups, dchunk, rnd); break;
    default: launch_k1<0, 0>(gwc, nhwc, grd, st, f, proj, depth_values, cost, V, C, D, h, w, num_groups, dchunk, rnd); break;
  }
  return after_launch("warp_cost");
}

// 16-byte vectors: the features, and a channels-last output.
extern "C" int casmvs_homo_warp_fwd(const float* src_feat, int feat_layout, const float* proj,
                                    const float* depth_values, float* warped, int out_layout,
                                    int B, int C, int D, int h, int w, void* stream) {
  CASMVS_REQUIRE_ALIGNED("homo_warp", src_feat, 16);
  if (out_layout == CASMVS_NHWC) CASMVS_REQUIRE_ALIGNED("homo_warp", warped, 16);
  CASMVS_REQUIRE(src_feat && proj && depth_values && warped, "homo_warp: null pointer");
  CASMVS_REQUIRE(feat_layout == CASMVS_NHWC,
                 "homo_warp: features must be channels-last (use casmvs_nchw_to_nhwc)");
  CASMVS_REQUIRE(C % kCPT == 0 && B >= 0 && B <= 65535 && D > 0 && h > 0 && w > 0,
                 "homo_warp: bad dims");
  CASMVS_REQUIRE((size_t)h * w * C < (1u << 31), "homo_warp: view too large");
  if (B == 0) return 0;
  const long threads = (long)h * w * (C / kCPT);
  dim3 grd((unsigned)((threads + kK1Threads - 1) / kK1Threads), (unsigned)B);
  cudaStream_t st = as_stream(stream);
  if (out_layout == CASMVS_NHWC)
    homo_warp_kernel<true><<<grd, kK1Threads, 0, st>>>(src_feat, proj, depth_values, warped, C, D, h, w);
  else
    homo_warp_kernel<false><<<grd, kK1Threads, 0, st>>>(src_feat, proj, depth_values, warped, C, D, h, w);
  return after_launch("homo_warp");
}

extern "C" int casmvs_nchw_to_nhwc(const float* in, float* out, int N, int C, size_t S,
                                   void* stream) {
  CASMVS_REQUIRE(in && out, "nchw_to_nhwc: null pointer");
  return launch_transpose(in, out, N, (size_t)C, S, as_stream(stream), "nchw_to_nhwc");
}

extern "C" int casmvs_nhwc_to_nchw(const float* in, float* out, int N, int C, size_t S,
                                   void* stream) {
  CASMVS_REQUIRE(in && out, "nhwc_to_nchw: null pointer");
  // (N,S,C) -> (N,C,S): same kernel with rows = S, cols = C
  return launch_transpose(in, out, N, S, (size_t)C, as_stream(stream), "nhwc_to_nchw");
}

extern "C" int casmvs_warp_cost_ladder_supported(int V, int C, int num_groups) {
  return warp_cost_staged(V, C, num_groups) != nullptr;
}

// Cascade-internal variant of casmvs_warp_cost_fwd: the hypotheses are the ladder
// first + step*d (see Hyp in k1_common.cuh) instead of a (B,D,h,w) tensor, or with
// CASMVS_INVERSE_DEPTH the inverse-depth ladder 1/(first - step*d).  The staged kernels
// read the features and write the cost volume (either layout) in 16-byte vectors.
extern "C" int casmvs_warp_cost_ladder_fwd(const float* feats, const float* proj,
                                           const float* first_map, const float* first_b,
                                           float first, const float* step_b, float step, float* cost,
                                           int round_tf32, int B, int V, int C, int D, int h, int w,
                                           int num_groups, void* stream) {
  CASMVS_REQUIRE_ALIGNED("warp_cost_ladder", feats, 16);
  CASMVS_REQUIRE_ALIGNED("warp_cost_ladder", cost, 16);
  CASMVS_REQUIRE(feats && proj && cost, "warp_cost_ladder: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && V >= 2 && C > 0 && D > 0 && h >= 2 && w >= 2,
                 "warp_cost_ladder: bad dims (h,w >= 2)");
  CASMVS_REQUIRE((size_t)h * w * C < (1u << 31), "warp_cost_ladder: view too large");
  if (B == 0) return 0;
  const StagedK1 run = warp_cost_staged(V, C, num_groups);
  CASMVS_REQUIRE(run, "warp_cost_ladder: shape not covered by the staged kernel "
                 "(casmvs_warp_cost_ladder_supported): materialise the hypotheses and call "
                 "casmvs_warp_cost_fwd (got V=%d C=%d G=%d)", V, C, num_groups);
  const int blocked = (round_tf32 & CASMVS_BLOCKED) ? 1 : 0;
  const int form = (round_tf32 & CASMVS_INVERSE_DEPTH) ? kLadderInverse : kLadderUniform;
  const int rnd = (round_tf32 & ~(CASMVS_BLOCKED | CASMVS_INVERSE_DEPTH)) ? 1 : 0;
  const Hyp hyp{nullptr, first_map, first_b, step_b, first, step};
  return run(feats, proj, hyp, cost, B, D, h, w, rnd, blocked, form, as_stream(stream));
}

// The per-pixel-step ladder of the adaptive mode (README "Adaptive depth ranges", regress.cu):
// plane d of pixel p is first_map[p] + step_map[p]*d, multiply and add each rounded.  Same
// coverage, layouts and flags (1, CASMVS_BLOCKED) as casmvs_warp_cost_ladder_fwd.
extern "C" int casmvs_warp_cost_ladder_step_fwd(const float* feats, const float* proj,
                                                const float* first_map, const float* step_map,
                                                float* cost, int round_tf32, int B, int V, int C,
                                                int D, int h, int w, int num_groups, void* stream) {
  CASMVS_REQUIRE_ALIGNED("warp_cost_ladder_step", feats, 16);
  CASMVS_REQUIRE_ALIGNED("warp_cost_ladder_step", cost, 16);
  CASMVS_REQUIRE(feats && proj && cost && first_map && step_map,
                 "warp_cost_ladder_step: null pointer");
  CASMVS_REQUIRE(B >= 0 && B <= 65535 && V >= 2 && C > 0 && D > 0 && h >= 2 && w >= 2,
                 "warp_cost_ladder_step: bad dims (h,w >= 2)");
  CASMVS_REQUIRE((size_t)h * w * C < (1u << 31), "warp_cost_ladder_step: view too large");
  CASMVS_REQUIRE((round_tf32 & ~(1 | CASMVS_BLOCKED)) == 0, "warp_cost_ladder_step: bad flags");
  if (B == 0) return 0;
  const StagedK1 run = warp_cost_staged(V, C, num_groups);
  CASMVS_REQUIRE(run, "warp_cost_ladder_step: shape not covered by the staged kernel "
                 "(casmvs_warp_cost_ladder_supported): materialise the hypotheses and call "
                 "casmvs_warp_cost_fwd (got V=%d C=%d G=%d)", V, C, num_groups);
  const int blocked = (round_tf32 & CASMVS_BLOCKED) ? 1 : 0;
  const Hyp hyp{nullptr, first_map, nullptr, step_map, 0.f, 0.f};
  return run(feats, proj, hyp, cost, B, D, h, w, round_tf32 & 1, blocked, kLadderPixelStep,
             as_stream(stream));
}
