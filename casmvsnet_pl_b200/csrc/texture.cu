// Texture a mesh from its views: per-face view candidates against the views' visibility buffers,
// labels, their smoothing, the chart components, the charts' rectangles, the atlas fill and the
// per-corner UVs (casmvsnet_pl_b200/texture.py drives these; oracle/texture_oracle.py restates them
// in numpy, bit for bit).  include/casmvs.h states the rule.
//
// The visibility buffers are the triangle rasteriser's key buffers (render.cu,
// casmvs_render_mesh_keys) and vertices are projected by the same project() (render_common.cuh),
// so a face's samples meet the pixels it was drawn into.  Every float and double operation the
// oracle restates is explicitly rounded; each face's candidates are kept by its own thread, views
// in index order; the only atomics are integer atomicMin / atomicMax, whose result does not depend
// on the schedule.
#include "render_common.cuh"

namespace casmvs {

constexpr int kTexK = 4;                      // candidates kept per face
constexpr int kTexPad = 2;                    // border of a vertex in its view, and of a rectangle
constexpr double kTexMinCos = 0.1;
constexpr float kTexDepthScale = 1.01f;       // 1 + DEPTH_TOL
constexpr int kTexMaxBatch = 8;               // views per casmvs_texture_scores call
constexpr int kTexMaxSide = 16384;

struct TexView {
  float P[12];
  double eye[3];
  const unsigned long long* zbuf;
  int W, H, index;
};
struct TexBatch {
  TexView v[kTexMaxBatch];
  int n;
};

struct Dv { double x, y, z; };

__device__ __forceinline__ double dot3(Dv a, Dv b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}

__device__ __forceinline__ bool tex_cam(const float* P, RenderCam& c) {
#pragma unroll
  for (int r = 0; r < 12; ++r) c.P[r] = P[r];
  return true;
}

// nearest pixel of (u, v) passes the depth test against zbuf
__device__ __forceinline__ bool tex_visible(const unsigned long long* zb, int W, float u, float v,
                                            float w) {
  const int px = (int)rintf(u), py = (int)rintf(v);
  const unsigned long long k = zb[(size_t)py * W + px];
  if (k == kKeyEmpty) return false;
  return w <= __fmul_rn(__uint_as_float((unsigned)(k >> 32)), kTexDepthScale);
}

__global__ void __launch_bounds__(256)
texture_scores_kernel(const __grid_constant__ TexBatch B, const float* __restrict__ verts,
                      const int* __restrict__ faces, int F, float* __restrict__ cand_score,
                      int* __restrict__ cand_view) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  float x[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int i = __ldg(faces + (size_t)f * 3 + k);
#pragma unroll
    for (int a = 0; a < 3; ++a) x[k][a] = __ldg(verts + (size_t)i * 3 + a);
  }
  const Dv e1{__dsub_rn(x[1][0], x[0][0]), __dsub_rn(x[1][1], x[0][1]), __dsub_rn(x[1][2], x[0][2])};
  const Dv e2{__dsub_rn(x[2][0], x[0][0]), __dsub_rn(x[2][1], x[0][1]), __dsub_rn(x[2][2], x[0][2])};
  const Dv n{__dsub_rn(__dmul_rn(e1.y, e2.z), __dmul_rn(e1.z, e2.y)),
             __dsub_rn(__dmul_rn(e1.z, e2.x), __dmul_rn(e1.x, e2.z)),
             __dsub_rn(__dmul_rn(e1.x, e2.y), __dmul_rn(e1.y, e2.x))};
  const double nn = dot3(n, n);
  if (!(nn > 0.0)) return;
  const double cd[3] = {
      __ddiv_rn(__dadd_rn(__dadd_rn(x[0][0], x[1][0]), x[2][0]), 3.0),
      __ddiv_rn(__dadd_rn(__dadd_rn(x[0][1], x[1][1]), x[2][1]), 3.0),
      __ddiv_rn(__dadd_rn(__dadd_rn(x[0][2], x[1][2]), x[2][2]), 3.0)};
  float cf[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    cf[a] = __fdiv_rn(__fadd_rn(__fadd_rn(x[0][a], x[1][a]), x[2][a]), 3.f);
  float sc[kTexK];
  int vw[kTexK];
#pragma unroll
  for (int j = 0; j < kTexK; ++j) {
    sc[j] = cand_score[(size_t)f * kTexK + j];
    vw[j] = cand_view[(size_t)f * kTexK + j];
  }
  bool changed = false;
  for (int b = 0; b < B.n; ++b) {
    const TexView& V = B.v[b];
    RenderCam cam;
    tex_cam(V.P, cam);
    float u[4], v[4], w[4];
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) ok = ok && project(cam, x[k][0], x[k][1], x[k][2], u[k], v[k], w[k]);
    ok = ok && project(cam, cf[0], cf[1], cf[2], u[3], v[3], w[3]);
    if (!ok) continue;
    const float ux = (float)(V.W - 1 - kTexPad), vy = (float)(V.H - 1 - kTexPad);
#pragma unroll
    for (int k = 0; k < 3; ++k)
      ok = ok && u[k] >= (float)kTexPad && u[k] <= ux && v[k] >= (float)kTexPad && v[k] <= vy;
    if (!ok) continue;
    const Dv d{__dsub_rn(cd[0], V.eye[0]), __dsub_rn(cd[1], V.eye[1]), __dsub_rn(cd[2], V.eye[2])};
    const double lhs = fabs(dot3(n, d));
    const double rhs = __dmul_rn(kTexMinCos, __dmul_rn(__dsqrt_rn(nn), __dsqrt_rn(dot3(d, d))));
    if (!(lhs >= rhs)) continue;
#pragma unroll
    for (int k = 0; k < 4; ++k) ok = ok && tex_visible(V.zbuf, V.W, u[k], v[k], w[k]);
    if (!ok) continue;
    const double a = __dsub_rn(__dmul_rn(__dsub_rn(u[1], u[0]), __dsub_rn(v[2], v[0])),
                               __dmul_rn(__dsub_rn(v[1], v[0]), __dsub_rn(u[2], u[0])));
    const float s = __double2float_rn(__dmul_rn(0.5, fabs(a)));
    // (score desc, view asc): views arrive in index order, so an equal score goes behind
    int pos = kTexK;
#pragma unroll
    for (int j = kTexK - 1; j >= 0; --j)
      if (vw[j] < 0 || s > sc[j]) pos = j;
    if (pos == kTexK) continue;
#pragma unroll
    for (int j = kTexK - 1; j > 0; --j)
      if (j > pos) { sc[j] = sc[j - 1]; vw[j] = vw[j - 1]; }
#pragma unroll
    for (int j = 0; j < kTexK; ++j)
      if (j == pos) { sc[j] = s; vw[j] = V.index; }
    changed = true;
  }
  if (changed) {
#pragma unroll
    for (int j = 0; j < kTexK; ++j) {
      cand_score[(size_t)f * kTexK + j] = sc[j];
      cand_view[(size_t)f * kTexK + j] = vw[j];
    }
  }
}

// One Jacobi round: f takes L when >= 2 of its manifold neighbours held L and L is a candidate of
// f scoring >= 0.5 x f's best; otherwise it keeps its label.
__global__ void __launch_bounds__(256)
texture_smooth_kernel(const int* __restrict__ nbr, const float* __restrict__ cand_score,
                      const int* __restrict__ cand_view, int F, const int* __restrict__ lin,
                      int* __restrict__ lout) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int l[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int g = __ldg(nbr + (size_t)f * 3 + k);
    l[k] = g >= 0 ? __ldg(lin + g) : -1;
  }
  int L = -1;
  if (l[0] >= 0 && (l[0] == l[1] || l[0] == l[2])) L = l[0];
  else if (l[1] >= 0 && l[1] == l[2]) L = l[1];
  int out = __ldg(lin + f);
  if (L >= 0) {
    const float thr = __fmul_rn(0.5f, __ldg(cand_score + (size_t)f * kTexK));
#pragma unroll
    for (int j = 0; j < kTexK; ++j)
      if (__ldg(cand_view + (size_t)f * kTexK + j) == L && __ldg(cand_score + (size_t)f * kTexK + j) >= thr)
        out = L;
  }
  lout[f] = out;
}

__global__ void __launch_bounds__(256) texture_iota_kernel(int* __restrict__ comp, int F) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F) comp[f] = f;
}

// Hook: across a manifold edge of equal labels >= 0, both faces and the larger root take the
// smaller component id.
__global__ void __launch_bounds__(256)
texture_hook_kernel(const int* __restrict__ nbr, const int* __restrict__ label, int F,
                    int* __restrict__ comp, unsigned* __restrict__ changed) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int L = __ldg(label + f);
  if (L < 0) return;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int g = __ldg(nbr + (size_t)f * 3 + k);
    if (g < 0 || __ldg(label + g) != L) continue;
    const int a = *(volatile int*)(comp + f), b = *(volatile int*)(comp + g);
    if (a == b) continue;
    const int lo = min(a, b), hi = max(a, b);
    atomicMin(comp + hi, lo);
    atomicMin(comp + f, lo);
    atomicMin(comp + g, lo);
    *changed = 1u;
  }
}

// Pointer jumping: every face points at the root of its current tree.
__global__ void __launch_bounds__(256) texture_jump_kernel(int* __restrict__ comp, int F) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int c = *(volatile int*)(comp + f);
  for (int n; (n = *(volatile int*)(comp + c)) < c;) c = n;
  atomicMin(comp + f, c);
}

__global__ void __launch_bounds__(256)
texture_rect_init_kernel(int* __restrict__ rect, int F) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  rect[(size_t)f * 4] = INT_MAX; rect[(size_t)f * 4 + 1] = INT_MAX;
  rect[(size_t)f * 4 + 2] = INT_MIN; rect[(size_t)f * 4 + 3] = INT_MIN;
}

__global__ void __launch_bounds__(256)
texture_rects_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                     const int* __restrict__ label, const int* __restrict__ comp,
                     const float* __restrict__ Ps, int* __restrict__ rect) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int L = __ldg(label + f);
  if (L < 0) return;
  RenderCam cam;
  tex_cam(Ps + (size_t)L * 16, cam);
  float lu = INFINITY, hu = -INFINITY, lv = INFINITY, hv = -INFINITY;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int i = __ldg(faces + (size_t)f * 3 + k);
    float u, v, w;
    project(cam, __ldg(verts + (size_t)i * 3), __ldg(verts + (size_t)i * 3 + 1),
            __ldg(verts + (size_t)i * 3 + 2), u, v, w);
    lu = fminf(lu, u); hu = fmaxf(hu, u); lv = fminf(lv, v); hv = fmaxf(hv, v);
  }
  int* r = rect + (size_t)__ldg(comp + f) * 4;
  atomicMin(r, (int)floorf(lu) - kTexPad);
  atomicMin(r + 1, (int)floorf(lv) - kTexPad);
  atomicMax(r + 2, (int)ceilf(hu) + kTexPad);
  atomicMax(r + 3, (int)ceilf(hv) + kTexPad);
}

// chart rows (9 int32): root face, view (-1 flat), x0, y0, x1, y1, page, ox, oy
__global__ void __launch_bounds__(256)
texture_fill_kernel(const int* __restrict__ charts, const unsigned long long* __restrict__ images,
                    const int* __restrict__ wh, const unsigned char* __restrict__ colours,
                    const int* __restrict__ faces, int S, unsigned char* __restrict__ atlas) {
  const int* c = charts + (size_t)blockIdx.x * 9;
  const int root = c[0], view = c[1], page = c[6], ox = c[7], oy = c[8];
  unsigned char* A = atlas + (size_t)page * S * S * 3;
  if (view < 0) {
    if (threadIdx.x >= 16) return;
    const int tx = threadIdx.x & 3, ty = threadIdx.x >> 2;
    unsigned char* d = A + ((size_t)(oy + ty) * S + ox + tx) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      int s = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) s += __ldg(colours + (size_t)__ldg(faces + (size_t)root * 3 + k) * 3 + ch);
      d[ch] = (unsigned char)((s + 1) / 3);     // s / 3 rounded: a third is never a half
    }
    return;
  }
  const unsigned char* src = reinterpret_cast<const unsigned char*>(images[view]);
  const int Wv = wh[view * 2];
  const int x0 = c[2], y0 = c[3], bw = c[4] - c[2] + 1, bh = c[5] - c[3] + 1;
  const long long n = (long long)bw * bh * 3;
  for (long long k = threadIdx.x; k < n; k += blockDim.x) {
    const int ch = (int)(k % 3);
    const long long t = k / 3;
    const int ty = (int)(t / bw), tx = (int)(t - (long long)ty * bw);
    A[((size_t)(oy + ty) * S + ox + tx) * 3 + ch] = src[((size_t)(y0 + ty) * Wv + x0 + tx) * 3 + ch];
  }
}

__global__ void __launch_bounds__(256)
texture_uvs_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                   const int* __restrict__ label, const int* __restrict__ slot,
                   const int* __restrict__ charts, const float* __restrict__ Ps, int S,
                   float* __restrict__ uv, int* __restrict__ page) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int* c = charts + (size_t)__ldg(slot + f) * 9;
  const int L = __ldg(label + f);
  const double Sd = (double)S;
  page[f] = c[6];
  if (L < 0) {
    // flat: corners at texel centres (1.5, 1.5), (2.5, 1.5), (1.5, 2.5) of the 4 x 4 square
    const double cx[3] = {1.5, 2.5, 1.5}, cy[3] = {1.5, 1.5, 2.5};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      uv[(size_t)f * 6 + 2 * k] = __double2float_rn(__ddiv_rn(__dadd_rn((double)c[7], cx[k]), Sd));
      uv[(size_t)f * 6 + 2 * k + 1] =
          __double2float_rn(__dsub_rn(1.0, __ddiv_rn(__dadd_rn((double)c[8], cy[k]), Sd)));
    }
    return;
  }
  RenderCam cam;
  tex_cam(Ps + (size_t)L * 16, cam);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int i = __ldg(faces + (size_t)f * 3 + k);
    float u, v, w;
    project(cam, __ldg(verts + (size_t)i * 3), __ldg(verts + (size_t)i * 3 + 1),
            __ldg(verts + (size_t)i * 3 + 2), u, v, w);
    const double a = __dadd_rn(__dadd_rn(__dsub_rn((double)u, (double)c[2]), (double)c[7]), 0.5);
    const double b = __dadd_rn(__dadd_rn(__dsub_rn((double)v, (double)c[3]), (double)c[8]), 0.5);
    uv[(size_t)f * 6 + 2 * k] = __double2float_rn(__ddiv_rn(a, Sd));
    uv[(size_t)f * 6 + 2 * k + 1] = __double2float_rn(__dsub_rn(1.0, __ddiv_rn(b, Sd)));
  }
}

inline unsigned tex_blocks(long long n) { return (unsigned)((n + 255) / 256); }

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_texture_scores(const float* verts, const int* faces, int F, int n_views,
                                     const float* P, const double* eye, const int* wh,
                                     const int* view_index, unsigned long long* const* zbufs,
                                     float* cand_score, int* cand_view, void* stream) {
  const char* what = "texture_scores";
  CASMVS_REQUIRE(F >= 0 && n_views >= 0 && n_views <= kTexMaxBatch,
                 "%s: need F >= 0 and 0 <= n_views <= %d (got %d, %d)", what, kTexMaxBatch, F,
                 n_views);
  CASMVS_REQUIRE(F == 0 || n_views == 0 || (verts && faces && cand_score && cand_view && P && eye &&
                                            wh && view_index && zbufs), "%s: null pointer", what);
  if (F == 0 || n_views == 0) return 0;
  TexBatch B;
  B.n = n_views;
  for (int j = 0; j < n_views; ++j) {
    for (int r = 0; r < 12; ++r) B.v[j].P[r] = P[j * 16 + r];
    for (int a = 0; a < 3; ++a) B.v[j].eye[a] = eye[j * 3 + a];
    B.v[j].W = wh[2 * j];
    B.v[j].H = wh[2 * j + 1];
    B.v[j].index = view_index[j];
    B.v[j].zbuf = zbufs[j];
    CASMVS_REQUIRE(B.v[j].W > 2 * kTexPad && B.v[j].H > 2 * kTexPad && B.v[j].W <= kTexMaxSide &&
                   B.v[j].H <= kTexMaxSide && zbufs[j], "%s: view %d: bad size %d x %d or null "
                   "key buffer", what, view_index[j], B.v[j].W, B.v[j].H);
  }
  texture_scores_kernel<<<tex_blocks(F), 256, 0, as_stream(stream)>>>(B, verts, faces, F, cand_score,
                                                                      cand_view);
  return after_launch(what);
}

extern "C" int casmvs_texture_smooth(const int* nbr, const float* cand_score, const int* cand_view,
                                     int F, const int* label_in, int* label_out, void* stream) {
  const char* what = "texture_smooth";
  CASMVS_REQUIRE(F >= 0, "%s: F < 0", what);
  if (F == 0) return 0;
  CASMVS_REQUIRE(nbr && cand_score && cand_view && label_in && label_out && label_in != label_out,
                 "%s: null or aliased pointer", what);
  texture_smooth_kernel<<<tex_blocks(F), 256, 0, as_stream(stream)>>>(nbr, cand_score, cand_view, F,
                                                                      label_in, label_out);
  return after_launch(what);
}

extern "C" int casmvs_texture_charts(const int* nbr, const int* label, int F, int* comp,
                                     unsigned* flag, int* rounds, void* stream) {
  const char* what = "texture_charts";
  CASMVS_REQUIRE(F >= 0, "%s: F < 0", what);
  CASMVS_REQUIRE(nbr && label && comp && flag && rounds, "%s: null pointer", what);
  *rounds = 0;
  if (F == 0) return 0;
  cudaStream_t st = as_stream(stream);
  texture_iota_kernel<<<tex_blocks(F), 256, 0, st>>>(comp, F);
  int rc = after_launch(what);
  if (rc) return rc;
  for (int it = 0; it <= F; ++it) {
    cudaError_t e = cudaMemsetAsync(flag, 0, sizeof(unsigned), st);
    CASMVS_REQUIRE(e == cudaSuccess, "%s: memset failed: %s", what, cudaGetErrorString(e));
    texture_hook_kernel<<<tex_blocks(F), 256, 0, st>>>(nbr, label, F, comp, flag);
    if ((rc = after_launch(what))) return rc;
    texture_jump_kernel<<<tex_blocks(F), 256, 0, st>>>(comp, F);
    if ((rc = after_launch(what))) return rc;
    unsigned changed = 0;
    e = cudaMemcpyAsync(&changed, flag, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    CASMVS_REQUIRE(e == cudaSuccess, "%s: %s", what, cudaGetErrorString(e));
    *rounds = it + 1;
    if (!changed) return 0;
  }
  CASMVS_REQUIRE(false, "%s: no convergence after %d rounds", what, F + 1);
}

extern "C" int casmvs_texture_rects(const float* verts, const int* faces, int F, const int* label,
                                    const int* comp, const float* Ps, int* rect, void* stream) {
  const char* what = "texture_rects";
  CASMVS_REQUIRE(F >= 0, "%s: F < 0", what);
  if (F == 0) return 0;
  CASMVS_REQUIRE(verts && faces && label && comp && Ps && rect, "%s: null pointer", what);
  cudaStream_t st = as_stream(stream);
  texture_rect_init_kernel<<<tex_blocks(F), 256, 0, st>>>(rect, F);
  const int rc = after_launch(what);
  if (rc) return rc;
  texture_rects_kernel<<<tex_blocks(F), 256, 0, st>>>(verts, faces, F, label, comp, Ps, rect);
  return after_launch(what);
}

extern "C" int casmvs_texture_fill(const int* charts, int n_charts, const unsigned long long* images,
                                   const int* wh, const unsigned char* colours, const int* faces,
                                   int S, unsigned char* atlas, void* stream) {
  const char* what = "texture_fill";
  CASMVS_REQUIRE(n_charts >= 0 && S >= 4 && S <= kTexMaxSide, "%s: need n_charts >= 0 and S in "
                 "4..%d (got %d, %d)", what, kTexMaxSide, n_charts, S);
  if (n_charts == 0) return 0;
  CASMVS_REQUIRE(charts && colours && faces && atlas, "%s: null pointer", what);
  texture_fill_kernel<<<n_charts, 256, 0, as_stream(stream)>>>(charts, images, wh, colours, faces,
                                                               S, atlas);
  return after_launch(what);
}

extern "C" int casmvs_texture_uvs(const float* verts, const int* faces, int F, const int* label,
                                  const int* slot, const int* charts, const float* Ps, int S,
                                  float* uv, int* page, void* stream) {
  const char* what = "texture_uvs";
  CASMVS_REQUIRE(F >= 0 && S >= 4 && S <= kTexMaxSide, "%s: need F >= 0 and S in 4..%d", what,
                 kTexMaxSide);
  if (F == 0) return 0;
  CASMVS_REQUIRE(verts && faces && label && slot && charts && Ps && uv && page, "%s: null pointer",
                 what);
  texture_uvs_kernel<<<tex_blocks(F), 256, 0, as_stream(stream)>>>(verts, faces, F, label, slot,
                                                                    charts, Ps, S, uv, page);
  return after_launch(what);
}
