// The world -> pixel projection and the empty key of the triangle rasteriser (render.cu), shared
// with the mesh texturing kernels (texture.cu) so that both see a vertex at the same (u, v, w).
#pragma once
#include "common.cuh"

namespace casmvs {

constexpr unsigned long long kKeyEmpty = ~0ull;

struct RenderCam {
  float P[12];                                // rows 0..2 of the world -> pixel matrix
  float eye[3];                               // camera centre, for the mesh shade
};

// ((A0 X + A1 Y) + A2 Z) + A3
__device__ __forceinline__ float proj_row(const float* A, float X, float Y, float Z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A[0], X), __fmul_rn(A[1], Y)), __fmul_rn(A[2], Z)),
                   A[3]);
}

// World point -> (u, v, w); false unless it is finite with w > 0 and finite u, v.
__device__ __forceinline__ bool project(const RenderCam& c, float X, float Y, float Z, float& u,
                                        float& v, float& w) {
  if (!(isfinite(X) && isfinite(Y) && isfinite(Z))) return false;
  w = proj_row(c.P + 8, X, Y, Z);
  if (!(w > 0.f) || !isfinite(w)) return false;
  u = __fdiv_rn(proj_row(c.P, X, Y, Z), w);
  v = __fdiv_rn(proj_row(c.P + 4, X, Y, Z), w);
  return isfinite(u) && isfinite(v);
}

}  // namespace casmvs
