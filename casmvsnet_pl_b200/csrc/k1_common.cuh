// Device helpers shared by the K1 kernels (warp_cost.cu: the gather kernel;
// warp_cost_smem.cu: the TMA-staged kernels).
#pragma once
#include "common.cuh"

namespace casmvs {

constexpr int kCPT = 8;          // channels per thread

// ---- fp32 pair helpers: two values in one 64-bit register (32-byte texel loads / stores);
// the arithmetic is one IEEE fp32 operation per lane, round to nearest -----------------
typedef unsigned long long u64;
__device__ __forceinline__ u64 pk2(float lo, float hi) {
  u64 r; asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "f"(lo), "f"(hi)); return r;
}
__device__ __forceinline__ void unpk2(u64 v, float& lo, float& hi) {
  asm("mov.b64 {%0,%1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
  float a0, a1, b0, b1, c0, c1;
  unpk2(a, a0, a1); unpk2(b, b0, b1); unpk2(c, c0, c1);
  return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  unpk2(a, a0, a1); unpk2(b, b0, b1);
  return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  unpk2(a, a0, a1); unpk2(b, b0, b1);
  return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
struct Tex8 { u64 v[4]; };   // 8 channels of one texel, as 4 packed pairs
__device__ __forceinline__ Tex8 ldg256(const float* p) {   // 32-byte aligned: two 16-byte loads
  Tex8 t;
  asm volatile("ld.global.nc.v2.b64 {%0,%1}, [%2];" : "=l"(t.v[0]), "=l"(t.v[1]) : "l"(p));
  asm volatile("ld.global.nc.v2.b64 {%0,%1}, [%2];" : "=l"(t.v[2]), "=l"(t.v[3]) : "l"(p + 4));
  return t;
}
__device__ __forceinline__ void stg256(float* p, const u64 (&v)[4]) {
  asm volatile("st.global.v2.b64 [%0], {%1,%2};" ::"l"(p), "l"(v[0]), "l"(v[1]) : "memory");
  asm volatile("st.global.v2.b64 [%0], {%1,%2};" ::"l"(p + 4), "l"(v[2]), "l"(v[3]) : "memory");
}
// The same 8 channels as two channel quads qstride floats apart: 4 for a channels-last volume,
// D*h*w*4 for one blocked by channel quads (B, C/4, D, h, w, 4).
__device__ __forceinline__ void stg256q(float* p, size_t qstride, const u64 (&v)[4]) {
  asm volatile("st.global.v2.b64 [%0], {%1,%2};" ::"l"(p), "l"(v[0]), "l"(v[1]) : "memory");
  asm volatile("st.global.v2.b64 [%0], {%1,%2};" ::"l"(p + qstride), "l"(v[2]), "l"(v[3]) : "memory");
}

__device__ __forceinline__ float round_tf32_f(float x) {
  uint32_t r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x)); return __uint_as_float(r);
}
__device__ __forceinline__ float rcp_approx(float x) {
  float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
}


// The kernel is instruction-issue bound rather than DRAM bound, so the sampler is written for
// instruction count:
//  * the 2x2 window is addressed as ONE base (clamped to [0,w-2]x[0,h-2]) plus
//    compile-time offsets {0, C, w*C, w*C + C}; the zero-padding rule of
//    grid_sample becomes a remap of the four weights at the image border,
//  * reciprocals are MUFU.RCP (1 ulp) instead of the IEEE sequence,
//  * the blend runs on fp32 pairs loaded as two 16-byte texel loads.
struct Window {
  Tex8 t00, t01, t10, t11;
};

// Bilinear blend of 8 channels, tap order nw, ne, sw, se like ATen grid_sampler_2d.  out(k, r)
// takes channel pair k as soon as it is blended: the gather kernel accumulates it right there,
// which keeps its register allocation (blending all four pairs first made it spill more).
template <class Out>
__device__ __forceinline__ void blend(const Window& win, float w00, float w01, float w10, float w11,
                                      Out&& out) {
  const u64 p00 = pk2(w00, w00), p01 = pk2(w01, w01), p10 = pk2(w10, w10), p11 = pk2(w11, w11);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    u64 a = mul2(win.t00.v[k], p00);
    a = fma2(win.t01.v[k], p01, a);
    a = fma2(win.t10.v[k], p10, a);
    out(k, fma2(win.t11.v[k], p11, a));
  }
}

// One sample of 8 channels gathered from the channels-last view at vbase (channel c0 already
// added).  Branch-free: a sample that contributes nothing (behind the camera / fully outside
// the source image) gets four zero weights and a clamped, always-valid address, so
// the loop body is straight-line code and ptxas can keep the loads of all views in
// flight at once.  CT = compile-time channel count (0: use C).
template <int CT, class Out>
__device__ __forceinline__ void gather_sample(const float* __restrict__ vbase, float qx, float qy,
                                              float qz, int h, int w, int C, int row_floats,
                                              Out&& out) {
  const float rz = rcp_approx(qz);
  const float u = qx * rz, v = qy * rz;
  const float x0f = floorf(u), y0f = floorf(v);
  // float->int saturates, so huge |u| fails the range test like ATen's within_bounds;
  // q_z <= 1e-7 is mapped to (w,h) = fully outside by the reference (modules.py:76-79)
  const int x0 = __float2int_rd(u), y0 = __float2int_rd(v);
  const bool valid = (qz > 1e-7f) && (unsigned)(x0 + 1) <= (unsigned)w &&
                     (unsigned)(y0 + 1) <= (unsigned)h;
  const float fx = u - x0f, fy = v - y0f;
  float wxa = 1.f - fx, wxb = fx, wya = 1.f - fy, wyb = fy;
  // border: texel x0 (or x0+1) is outside => its weight is dropped; the pair
  // (xs, xs+1) stays inside the image and the surviving weight moves to its slot
  if (x0 < 0) { wxa = wxb; wxb = 0.f; }
  if (x0 > w - 2) { wxb = wxa; wxa = 0.f; }
  if (y0 < 0) { wya = wyb; wyb = 0.f; }
  if (y0 > h - 2) { wyb = wya; wya = 0.f; }
  if (!valid) { wxa = 0.f; wxb = 0.f; }
  const int xs = min(max(x0, 0), w - 2), ys = min(max(y0, 0), h - 2);
  const float w00 = wxa * wya, w01 = wxb * wya, w10 = wxa * wyb, w11 = wxb * wyb;
  const int cc = CT > 0 ? CT : C;
  const unsigned off = (unsigned)(ys * row_floats + xs * cc);
  const float* p = vbase + off;
  Window win;
  win.t00 = ldg256(p);
  win.t01 = ldg256(p + cc);
  win.t10 = ldg256(p + row_floats);
  win.t11 = ldg256(p + row_floats + cc);
  blend(win, w00, w01, w10, w11, out);
}

// Variance cost of 8 channels from the sums S and Q of the V views: Q/V - (S/V)^2
// (mvsnet.py:166-168), inv_v2 = (1/V, 1/V), ninv_v2 = -inv_v2.  round_tf32: the tensor-core conv
// reads fp32 bits as tf32 by truncation; rounding here keeps the next layer's operand unbiased
// (round-to-nearest instead of toward zero).
__device__ __forceinline__ void variance(const u64 (&S)[4], const u64 (&Q)[4], u64 inv_v2,
                                         u64 ninv_v2, int round_tf32, u64 (&o)[4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const u64 m = mul2(S[k], inv_v2), mn = mul2(S[k], ninv_v2);
    o[k] = fma2(mn, m, mul2(Q[k], inv_v2));
  }
  if (round_tf32) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float lo, hi;
      unpk2(o[k], lo, hi);
      o[k] = pk2(round_tf32_f(lo), round_tf32_f(hi));
    }
  }
}


// Where a pixel's depth hypotheses come from: the (B,D,h,w) tensor of the public API, or -- in
// the cascade -- the ladder first + step*d that get_depth_values / the initial planes define
// (models/modules.py:44-48, models/mvsnet.py:215-229), generated in the kernel with the SAME two
// roundings (multiply, then add) so that the (B,D,h,w) tensor never has to exist in HBM.
struct Hyp {
  const float* dv;         // (B,D,h,w) or null => ladder
  const float* first_map;  // (B,h,w) first hypothesis per pixel, or null
  const float* first_b;    // (B) first hypothesis per batch item, or null
  const float* step_b;     // (B) plane spacing per batch item, or null
  float first, step;       // scalars used when the pointers above are null
};
struct HypPix {
  const float* p;
  size_t hw;
  float first, step;
  __device__ __forceinline__ HypPix(const Hyp& h, int b, int D, size_t hw_, int pix) : hw(hw_) {
    p = h.dv ? h.dv + (size_t)b * D * hw_ + pix : nullptr;
    first = h.first_map ? __ldg(h.first_map + (size_t)b * hw_ + pix) : h.first_b ? __ldg(h.first_b + b) : h.first;
    step = h.step_b ? __ldg(h.step_b + b) : h.step;
  }
  __device__ __forceinline__ float at(int d) const {
    return p ? __ldg(p + (size_t)d * hw) : __fadd_rn(first, __fmul_rn(step, (float)d));
  }
};

}  // namespace casmvs
