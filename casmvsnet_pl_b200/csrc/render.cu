// Headless rendering of point clouds and coloured triangle meshes into an image and a depth map
// (casmvsnet_pl_b200/render.py drives these; oracle/render_oracle.py restates them in numpy, bit
// for bit).
//
// Depth test: every covered pixel takes one 64-bit atomicMin of the key (float bits of the camera
// depth w > 0) << 32 | primitive index.  Positive floats order like their bits, so the nearest
// primitive wins and an exact tie goes to the lower index, whatever the thread schedule.  A
// resolve pass then turns each pixel's key into a colour and a depth; for triangles it
// re-evaluates the winner's interpolation at the pixel, so colours never race.
//
// All float arithmetic the oracle restates is explicitly rounded (no FMA contraction), in the
// order include/casmvs.h states.
//
// Triangles: one thread per triangle projects it and rasterises its screen bounding box when that
// is at most kSmallBox x kSmallBox pixels; larger boxes go to a list that whole CTAs work through,
// so a triangle filling the screen does not serialise in one thread.
#include "render_common.cuh"

namespace casmvs {

constexpr int kSmallBox = 8;                  // px per side rasterised by the triangle's thread
constexpr int kMaxSide = 16384, kMaxPointSize = 64;

__device__ __forceinline__ unsigned long long depth_key(float w, unsigned idx) {
  return ((unsigned long long)__float_as_uint(w) << 32) | idx;
}

__device__ __forceinline__ void depth_test(unsigned long long* zbuf, size_t pix,
                                           unsigned long long key) {
  // a plain read first: most losing fragments never issue the atomic
  if (key < *(volatile unsigned long long*)(zbuf + pix)) atomicMin(zbuf + pix, key);
}

// ---------------------------------------------------------------------------- points
__global__ void __launch_bounds__(256)
render_points_kernel(const __grid_constant__ RenderCam cam, const float* __restrict__ xyz,
                     unsigned long long n, int W, int H, int size,
                     unsigned long long* __restrict__ zbuf) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float u, v, w;
  if (!project(cam, __ldg(xyz + i * 3), __ldg(xyz + i * 3 + 1), __ldg(xyz + i * 3 + 2), u, v, w))
    return;
  // integer pixel centres in [u - s/2, u + s/2) x [v - s/2, v + s/2)
  const float h = 0.5f * (float)size;         // exact
  const float x0 = ceilf(__fsub_rn(u, h)), x1 = __fsub_rn(ceilf(__fadd_rn(u, h)), 1.f);
  const float y0 = ceilf(__fsub_rn(v, h)), y1 = __fsub_rn(ceilf(__fadd_rn(v, h)), 1.f);
  if (x1 < 0.f || y1 < 0.f || x0 > (float)(W - 1) || y0 > (float)(H - 1)) return;
  const int xa = (int)fmaxf(x0, 0.f), xb = (int)fminf(x1, (float)(W - 1));
  const int ya = (int)fmaxf(y0, 0.f), yb = (int)fminf(y1, (float)(H - 1));
  const unsigned long long key = depth_key(w, (unsigned)i);
  for (int y = ya; y <= yb; ++y)
    for (int x = xa; x <= xb; ++x) depth_test(zbuf, (size_t)y * W + x, key);
}

__global__ void __launch_bounds__(256)
render_points_resolve_kernel(const unsigned long long* __restrict__ zbuf,
                             const unsigned char* __restrict__ rgb, int npix,
                             unsigned char* __restrict__ image, float* __restrict__ depth) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const unsigned long long k = zbuf[p];
  unsigned char c[3] = {128, 128, 255};
  float d = 0.f;
  if (k != kKeyEmpty) {
    const size_t i = (unsigned)k;
    c[0] = __ldg(rgb + i * 3); c[1] = __ldg(rgb + i * 3 + 1); c[2] = __ldg(rgb + i * 3 + 2);
    d = __uint_as_float((unsigned)(k >> 32));
  }
  image[(size_t)p * 3] = c[0]; image[(size_t)p * 3 + 1] = c[1]; image[(size_t)p * 3 + 2] = c[2];
  depth[p] = d;
}

// ---------------------------------------------------------------------------- triangles
struct Tri {
  float u[3], v[3], w[3];
  int x0, x1, y0, y1;                         // clamped pixel bounding box (inclusive)
};

// (bx - ax)(py - ay) - (by - ay)(px - ax)
__device__ __forceinline__ float edge_fn(float ax, float ay, float bx, float by, float px, float py) {
  return __fsub_rn(__fmul_rn(__fsub_rn(bx, ax), __fsub_rn(py, ay)),
                   __fmul_rn(__fsub_rn(by, ay), __fsub_rn(px, ax)));
}

// Face t -> projected triangle with a non-empty on-screen box; false when it is skipped.  A face
// index outside [0, nv) raises *bad and reads nothing.
__device__ __forceinline__ bool setup_tri(const RenderCam& cam, const float* __restrict__ verts,
                                          int nv, const int* __restrict__ faces, unsigned t, int W,
                                          int H, Tri& T, unsigned* bad) {
  int f[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    f[k] = __ldg(faces + (size_t)t * 3 + k);
    if (f[k] < 0 || f[k] >= nv) {
      if (bad) atomicOr(bad, 1u);
      return false;
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float* p = verts + (size_t)f[k] * 3;
    if (!project(cam, __ldg(p), __ldg(p + 1), __ldg(p + 2), T.u[k], T.v[k], T.w[k])) return false;
  }
  const float area = edge_fn(T.u[0], T.v[0], T.u[1], T.v[1], T.u[2], T.v[2]);
  if (!(area != 0.f) || !isfinite(area)) return false;
  const float lx = ceilf(fminf(fminf(T.u[0], T.u[1]), T.u[2]));
  const float hx = floorf(fmaxf(fmaxf(T.u[0], T.u[1]), T.u[2]));
  const float ly = ceilf(fminf(fminf(T.v[0], T.v[1]), T.v[2]));
  const float hy = floorf(fmaxf(fmaxf(T.v[0], T.v[1]), T.v[2]));
  if (hx < 0.f || hy < 0.f || lx > (float)(W - 1) || ly > (float)(H - 1) || lx > hx || ly > hy)
    return false;
  T.x0 = (int)fmaxf(lx, 0.f); T.x1 = (int)fminf(hx, (float)(W - 1));
  T.y0 = (int)fmaxf(ly, 0.f); T.y1 = (int)fminf(hy, (float)(H - 1));
  return true;
}

// Edge functions at pixel centre (x, y): e0 of edge 1->2, e1 of 2->0, e2 of 0->1.  Covered when
// all are >= 0 or all <= 0; then q_k = e_k / w_k, den = (q0 + q1) + q2 and the depth is
// ((e0 + e1) + e2) / den (1/w interpolated linearly in screen space).
__device__ __forceinline__ bool tri_depth(const Tri& T, int x, int y, float q[3], float& den,
                                          float& w) {
  const float px = (float)x, py = (float)y;
  const float e0 = edge_fn(T.u[1], T.v[1], T.u[2], T.v[2], px, py);
  const float e1 = edge_fn(T.u[2], T.v[2], T.u[0], T.v[0], px, py);
  const float e2 = edge_fn(T.u[0], T.v[0], T.u[1], T.v[1], px, py);
  if (!((e0 >= 0.f && e1 >= 0.f && e2 >= 0.f) || (e0 <= 0.f && e1 <= 0.f && e2 <= 0.f)))
    return false;
  q[0] = __fdiv_rn(e0, T.w[0]); q[1] = __fdiv_rn(e1, T.w[1]); q[2] = __fdiv_rn(e2, T.w[2]);
  den = __fadd_rn(__fadd_rn(q[0], q[1]), q[2]);
  w = __fdiv_rn(__fadd_rn(__fadd_rn(e0, e1), e2), den);
  return w > 0.f && isfinite(w);
}

__device__ __forceinline__ void raster_px(const Tri& T, unsigned t, int x, int y, int W,
                                          unsigned long long* zbuf) {
  float q[3], den, w;
  if (tri_depth(T, x, y, q, den, w)) depth_test(zbuf, (size_t)y * W + x, depth_key(w, t));
}

// ws[0] = number of large triangles, ws[1] = bad-face flag, ws[2..] = their indices
__global__ void __launch_bounds__(256)
render_tris_kernel(const __grid_constant__ RenderCam cam, const float* __restrict__ verts, int nv,
                   const int* __restrict__ faces, int nf, int W, int H,
                   unsigned long long* __restrict__ zbuf, unsigned* __restrict__ ws) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nf) return;
  Tri T;
  if (!setup_tri(cam, verts, nv, faces, (unsigned)t, W, H, T, ws + 1)) return;
  if (T.x1 - T.x0 >= kSmallBox || T.y1 - T.y0 >= kSmallBox) {
    ws[2 + atomicAdd(ws, 1u)] = (unsigned)t;
    return;
  }
  for (int y = T.y0; y <= T.y1; ++y)
    for (int x = T.x0; x <= T.x1; ++x) raster_px(T, (unsigned)t, x, y, W, zbuf);
}

__global__ void __launch_bounds__(256)
render_big_tris_kernel(const __grid_constant__ RenderCam cam, const float* __restrict__ verts,
                       int nv, const int* __restrict__ faces, int W, int H,
                       unsigned long long* __restrict__ zbuf, const unsigned* __restrict__ ws) {
  const unsigned n = ws[0];
  for (unsigned j = blockIdx.x; j < n; j += gridDim.x) {
    const unsigned t = ws[2 + j];
    Tri T;
    if (!setup_tri(cam, verts, nv, faces, t, W, H, T, nullptr)) continue;   // cannot happen
    const int bw = T.x1 - T.x0 + 1;
    const long long npx = (long long)bw * (T.y1 - T.y0 + 1);
    for (long long k = threadIdx.x; k < npx; k += blockDim.x) {
      const int dy = (int)(k / bw);
      raster_px(T, t, T.x0 + (int)(k - (long long)dy * bw), T.y0 + dy, W, zbuf);
    }
  }
}

// Shade of face t: 0.3 + 0.7 min(1, |n.d| / (|n| |d|)), n = (v1 - v0) x (v2 - v0), d = centroid -
// eye; 0.3 when |n| |d| is 0.
__device__ __forceinline__ float face_shade(const RenderCam& cam, const float* a, const float* b,
                                            const float* c) {
  float e1[3], e2[3], d[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    e1[k] = __fsub_rn(b[k], a[k]);
    e2[k] = __fsub_rn(c[k], a[k]);
    d[k] = __fsub_rn(__fdiv_rn(__fadd_rn(__fadd_rn(a[k], b[k]), c[k]), 3.f), cam.eye[k]);
  }
  const float n0 = __fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1]));
  const float n1 = __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2]));
  const float n2 = __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0]));
  const float nn = __fadd_rn(__fadd_rn(__fmul_rn(n0, n0), __fmul_rn(n1, n1)), __fmul_rn(n2, n2));
  const float dd = __fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])),
                             __fmul_rn(d[2], d[2]));
  const float dot = __fadd_rn(__fadd_rn(__fmul_rn(n0, d[0]), __fmul_rn(n1, d[1])), __fmul_rn(n2, d[2]));
  const float den = __fmul_rn(__fsqrt_rn(nn), __fsqrt_rn(dd));
  float cs = __fdiv_rn(fabsf(dot), den);
  cs = (den > 0.f && isfinite(cs)) ? fminf(cs, 1.f) : 0.f;
  return __fadd_rn(0.3f, __fmul_rn(0.7f, cs));
}

__global__ void __launch_bounds__(256)
render_mesh_resolve_kernel(const __grid_constant__ RenderCam cam, const float* __restrict__ verts,
                           const unsigned char* __restrict__ colours, int nv,
                           const int* __restrict__ faces, const unsigned long long* __restrict__ zbuf,
                           int W, int H, unsigned char* __restrict__ image,
                           float* __restrict__ depth) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= W * H) return;
  const unsigned long long k = zbuf[p];
  unsigned char out[3] = {128, 128, 255};
  float d = 0.f;
  if (k != kKeyEmpty) {
    const unsigned t = (unsigned)k;
    d = __uint_as_float((unsigned)(k >> 32));
    Tri T;
    float q[3], den, w;
    // the pixel's winner passed both tests when it was rasterised; the same bits pass them again
    if (setup_tri(cam, verts, nv, faces, t, W, H, T, nullptr) && tri_depth(T, p % W, p / W, q, den, w)) {
      int f[3];
      float x[3][3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        f[j] = __ldg(faces + (size_t)t * 3 + j);
#pragma unroll
        for (int a = 0; a < 3; ++a) x[j][a] = __ldg(verts + (size_t)f[j] * 3 + a);
      }
      const float s = face_shade(cam, x[0], x[1], x[2]);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        float c[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) c[j] = (float)__ldg(colours + (size_t)f[j] * 3 + ch);
        const float num = __fadd_rn(__fadd_rn(__fmul_rn(q[0], c[0]), __fmul_rn(q[1], c[1])),
                                    __fmul_rn(q[2], c[2]));
        const float val = floorf(__fadd_rn(__fmul_rn(__fdiv_rn(num, den), s), 0.5f));
        out[ch] = (unsigned char)fminf(255.f, fmaxf(0.f, val));
      }
    }
  }
  image[(size_t)p * 3] = out[0]; image[(size_t)p * 3 + 1] = out[1]; image[(size_t)p * 3 + 2] = out[2];
  depth[p] = d;
}

// Textured resolve: the winner's UV interpolated perspective-correctly (as the colours above),
// then the page sampled bilinearly with texel centres at i + 0.5 and clamped indices.  Unshaded.
__global__ void __launch_bounds__(256)
render_textured_resolve_kernel(const __grid_constant__ RenderCam cam, const float* __restrict__ verts,
                               int nv, const int* __restrict__ faces, const float* __restrict__ uv,
                               const int* __restrict__ page, const unsigned char* __restrict__ atlas,
                               int n_pages, int S, const unsigned long long* __restrict__ zbuf,
                               int W, int H, unsigned char* __restrict__ image,
                               float* __restrict__ depth) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= W * H) return;
  const unsigned long long k = zbuf[p];
  unsigned char out[3] = {128, 128, 255};
  float d = 0.f;
  if (k != kKeyEmpty) {
    const unsigned t = (unsigned)k;
    d = __uint_as_float((unsigned)(k >> 32));
    Tri T;
    float q[3], den, w;
    const int pg = __ldg(page + t);
    if (pg >= 0 && pg < n_pages && setup_tri(cam, verts, nv, faces, t, W, H, T, nullptr) &&
        tri_depth(T, p % W, p / W, q, den, w)) {
      const float* c = uv + (size_t)t * 6;
      const float tu = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], __ldg(c)), __fmul_rn(q[1], __ldg(c + 2))),
                                           __fmul_rn(q[2], __ldg(c + 4))), den);
      const float tv = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], __ldg(c + 1)), __fmul_rn(q[1], __ldg(c + 3))),
                                           __fmul_rn(q[2], __ldg(c + 5))), den);
      const float Sf = (float)S;
      // texel space; clamped to [-1, S] first so that the integer conversion is defined
      const float x = fminf(fmaxf(__fsub_rn(__fmul_rn(tu, Sf), 0.5f), -1.f), Sf);
      const float y = fminf(fmaxf(__fsub_rn(__fmul_rn(__fsub_rn(1.f, tv), Sf), 0.5f), -1.f), Sf);
      const float fx = floorf(x), fy = floorf(y);
      const float ax = __fsub_rn(x, fx), ay = __fsub_rn(y, fy);
      const int x0 = min(max((int)fx, 0), S - 1), x1 = min(max((int)fx + 1, 0), S - 1);
      const int y0 = min(max((int)fy, 0), S - 1), y1 = min(max((int)fy + 1, 0), S - 1);
      const unsigned char* A = atlas + (size_t)pg * S * S * 3;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float c00 = (float)__ldg(A + ((size_t)y0 * S + x0) * 3 + ch);
        const float c10 = (float)__ldg(A + ((size_t)y0 * S + x1) * 3 + ch);
        const float c01 = (float)__ldg(A + ((size_t)y1 * S + x0) * 3 + ch);
        const float c11 = (float)__ldg(A + ((size_t)y1 * S + x1) * 3 + ch);
        const float r0 = __fadd_rn(__fmul_rn(__fsub_rn(1.f, ax), c00), __fmul_rn(ax, c10));
        const float r1 = __fadd_rn(__fmul_rn(__fsub_rn(1.f, ax), c01), __fmul_rn(ax, c11));
        const float val = floorf(__fadd_rn(__fadd_rn(__fmul_rn(__fsub_rn(1.f, ay), r0),
                                                     __fmul_rn(ay, r1)), 0.5f));
        out[ch] = (unsigned char)fminf(255.f, fmaxf(0.f, val));
      }
    }
  }
  image[(size_t)p * 3] = out[0]; image[(size_t)p * 3 + 1] = out[1]; image[(size_t)p * 3 + 2] = out[2];
  depth[p] = d;
}

inline unsigned render_blocks(unsigned long long n) { return (unsigned)((n + 255) / 256); }

inline RenderCam make_cam(const float* P, const float* eye) {
  RenderCam c;
  for (int r = 0; r < 12; ++r) c.P[r] = P[r];
  for (int a = 0; a < 3; ++a) c.eye[a] = eye ? eye[a] : 0.f;
  return c;
}

}  // namespace casmvs

using namespace casmvs;

#define RENDER_CHECK_SIZE(what, W, H)                                                       \
  CASMVS_REQUIRE((W) >= 1 && (W) <= kMaxSide && (H) >= 1 && (H) <= kMaxSide,                \
                 "%s: W and H must lie in 1..%d (got %d x %d)", what, kMaxSide, (W), (H))

extern "C" int casmvs_render_points_fwd(const float* xyz, const unsigned char* rgb, long long n,
                                        const float* P, int W, int H, int point_size,
                                        unsigned long long* zbuf, unsigned char* image,
                                        float* depth, void* stream) {
  const char* what = "render_points_fwd";
  CASMVS_REQUIRE(n >= 0 && n < (1ll << 32), "%s: need 0 <= n < 2^32 points (got %lld)", what, n);
  RENDER_CHECK_SIZE(what, W, H);
  CASMVS_REQUIRE(point_size >= 1 && point_size <= kMaxPointSize,
                 "%s: point_size must lie in 1..%d (got %d)", what, kMaxPointSize, point_size);
  CASMVS_REQUIRE_ALIGNED(what, xyz, 4);
  CASMVS_REQUIRE_ALIGNED(what, zbuf, 8);
  CASMVS_REQUIRE_ALIGNED(what, depth, 4);
  CASMVS_REQUIRE(P && zbuf && image && depth && (n == 0 || (xyz && rgb)), "%s: null pointer", what);
  const RenderCam cam = make_cam(P, nullptr);
  cudaStream_t st = as_stream(stream);
  const size_t npix = (size_t)W * H;
  cudaError_t e = cudaMemsetAsync(zbuf, 0xff, npix * sizeof(unsigned long long), st);
  CASMVS_REQUIRE(e == cudaSuccess, "%s: memset failed: %s", what, cudaGetErrorString(e));
  if (n > 0) {
    render_points_kernel<<<render_blocks(n), 256, 0, st>>>(cam, xyz, (unsigned long long)n, W, H,
                                                          point_size, zbuf);
    const int rc = after_launch(what);
    if (rc) return rc;
  }
  render_points_resolve_kernel<<<render_blocks(npix), 256, 0, st>>>(zbuf, rgb, (int)npix, image, depth);
  return after_launch(what);
}

extern "C" size_t casmvs_render_mesh_workspace_bytes(int n_faces) {
  return n_faces < 0 ? 0 : (size_t)(n_faces + 2) * sizeof(unsigned);
}

// The raster pass of a mesh: zbuf cleared, then every face's covered pixels keyed; the bad-face
// flag is read back (one synchronise).
static int raster_mesh(const char* what, const RenderCam& cam, const float* verts, int n_vertices,
                       const int* faces, int n_faces, int W, int H, unsigned long long* zbuf,
                       unsigned* ws, cudaStream_t st) {
  const size_t npix = (size_t)W * H;
  cudaError_t e = cudaMemsetAsync(zbuf, 0xff, npix * sizeof(unsigned long long), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(ws, 0, 2 * sizeof(unsigned), st);
  CASMVS_REQUIRE(e == cudaSuccess, "%s: memset failed: %s", what, cudaGetErrorString(e));
  if (n_faces > 0) {
    render_tris_kernel<<<render_blocks(n_faces), 256, 0, st>>>(cam, verts, n_vertices, faces,
                                                               n_faces, W, H, zbuf, ws);
    int rc = after_launch(what);
    if (rc) return rc;
    render_big_tris_kernel<<<num_sms() * 8, 256, 0, st>>>(cam, verts, n_vertices, faces, W, H,
                                                          zbuf, ws);
    rc = after_launch(what);
    if (rc) return rc;
    unsigned bad = 0;
    e = cudaMemcpyAsync(&bad, ws + 1, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    CASMVS_REQUIRE(e == cudaSuccess, "%s: %s", what, cudaGetErrorString(e));
    CASMVS_REQUIRE(!bad, "%s: a face index lies outside [0, %d)", what, n_vertices);
  }
  return 0;
}

#define RENDER_CHECK_MESH(what)                                                              \
  CASMVS_REQUIRE(n_vertices >= 0 && n_faces >= 0, "%s: negative vertex or face count", what); \
  RENDER_CHECK_SIZE(what, W, H);                                                              \
  CASMVS_REQUIRE_ALIGNED(what, verts, 4);                                                     \
  CASMVS_REQUIRE_ALIGNED(what, faces, 4);                                                     \
  CASMVS_REQUIRE_ALIGNED(what, zbuf, 8);                                                      \
  CASMVS_REQUIRE_ALIGNED(what, workspace, 4);                                                 \
  CASMVS_REQUIRE(workspace_bytes >= casmvs_render_mesh_workspace_bytes(n_faces),              \
                 "%s: workspace of %zu bytes, need %zu", what, workspace_bytes,               \
                 casmvs_render_mesh_workspace_bytes(n_faces))

extern "C" int casmvs_render_mesh_fwd(const float* verts, const unsigned char* colours, int n_vertices,
                                      const int* faces, int n_faces, const float* P, const float* eye,
                                      int W, int H, unsigned long long* zbuf, void* workspace,
                                      size_t workspace_bytes, unsigned char* image, float* depth,
                                      void* stream) {
  const char* what = "render_mesh_fwd";
  RENDER_CHECK_MESH(what);
  CASMVS_REQUIRE_ALIGNED(what, depth, 4);
  CASMVS_REQUIRE(P && eye && zbuf && workspace && image && depth &&
                 (n_faces == 0 || (verts && colours && faces)), "%s: null pointer", what);
  const RenderCam cam = make_cam(P, eye);
  cudaStream_t st = as_stream(stream);
  const size_t npix = (size_t)W * H;
  const int rc = raster_mesh(what, cam, verts, n_vertices, faces, n_faces, W, H, zbuf,
                             static_cast<unsigned*>(workspace), st);
  if (rc) return rc;
  render_mesh_resolve_kernel<<<render_blocks(npix), 256, 0, st>>>(cam, verts, colours, n_vertices,
                                                                  faces, zbuf, W, H, image, depth);
  return after_launch(what);
}

extern "C" int casmvs_render_mesh_keys(const float* verts, int n_vertices, const int* faces,
                                       int n_faces, const float* P, int W, int H,
                                       unsigned long long* zbuf, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  const char* what = "render_mesh_keys";
  RENDER_CHECK_MESH(what);
  CASMVS_REQUIRE(P && zbuf && workspace && (n_faces == 0 || (verts && faces)), "%s: null pointer",
                 what);
  return raster_mesh(what, make_cam(P, nullptr), verts, n_vertices, faces, n_faces, W, H, zbuf,
                     static_cast<unsigned*>(workspace), as_stream(stream));
}

extern "C" int casmvs_render_textured_mesh_fwd(const float* verts, int n_vertices, const int* faces,
                                               int n_faces, const float* uv, const int* page,
                                               const unsigned char* atlas, int n_pages, int S,
                                               const float* P, int W, int H,
                                               unsigned long long* zbuf, void* workspace,
                                               size_t workspace_bytes, unsigned char* image,
                                               float* depth, void* stream) {
  const char* what = "render_textured_mesh_fwd";
  RENDER_CHECK_MESH(what);
  CASMVS_REQUIRE_ALIGNED(what, uv, 4);
  CASMVS_REQUIRE_ALIGNED(what, page, 4);
  CASMVS_REQUIRE_ALIGNED(what, depth, 4);
  CASMVS_REQUIRE(n_pages >= 1 && S >= 1 && S <= kMaxSide, "%s: need n_pages >= 1 and S in 1..%d "
                 "(got %d, %d)", what, kMaxSide, n_pages, S);
  CASMVS_REQUIRE(P && zbuf && workspace && image && depth && atlas &&
                 (n_faces == 0 || (verts && faces && uv && page)), "%s: null pointer", what);
  const RenderCam cam = make_cam(P, nullptr);
  cudaStream_t st = as_stream(stream);
  const size_t npix = (size_t)W * H;
  const int rc = raster_mesh(what, cam, verts, n_vertices, faces, n_faces, W, H, zbuf,
                             static_cast<unsigned*>(workspace), st);
  if (rc) return rc;
  render_textured_resolve_kernel<<<render_blocks(npix), 256, 0, st>>>(
      cam, verts, n_vertices, faces, uv, page, atlas, n_pages, S, zbuf, W, H, image, depth);
  return after_launch(what);
}
