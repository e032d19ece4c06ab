// TSDF fusion of masked depth maps into a sparse voxel volume and marching-cubes extraction of a
// coloured triangle mesh (casmvsnet_pl_b200/mesh.py drives these; oracle/mesh_oracle.py restates
// them in numpy, bit for bit).
//
// Volume: bricks of 8^3 voxels, voxel ijk centred at ijk * voxel in world coordinates.  Brick
// (bx, by, bz) holds voxels i = 8 bx + lx, ... ; its key packs (b + 2^20) into 21 bits per axis,
// x highest, so sorted keys order bricks by (bx, by, bz).  Voxel v = 512 * brick + (lz * 8 + ly)
// * 8 + lx of the sorted brick list; tsdf, weight (a view count) and colour (3 floats) per voxel.
//
// Integration (Curless & Levoy's projective TSDF): one thread per voxel walks the views of a
// launch in order, so each voxel is read and written once per batch of kMeshViews views, and the
// result does not depend on scheduling (no atomics).  All float arithmetic is explicitly rounded
// (no FMA contraction), in the order casmvs.h states, so a float32 numpy restatement gives the
// same bits.
//
// Extraction: a cell is the cube of 8 voxel centres with lower corner v; it is meshed when all
// its corners are allocated and have weight > 0.  Pass 1 counts triangles per cell and flags the
// crossing edges those cells use (each voxel owns the +x, +y, +z edges leaving it); an integer
// scan of each (torch) gives vertex ids and triangle offsets; pass 2 writes the vertices (double
// interpolation, one rounding) and pass 3 the triangles, in cell order and table order.
#include "common.cuh"
#include "mc_table.h"

namespace casmvs {

constexpr int kMeshViews = 8;                 // views per integration launch
constexpr int kBias = 1 << 20;                // key offset per axis
constexpr int kBrickMin = -(1 << 20), kBrickMax = (1 << 20) - 2;
constexpr long long kMaxBricks = 0x7fffffffLL / (512 * 3);   // voxel edge ids fit an int
constexpr long long kKeyNone = 0x7fffffffffffffffLL;

struct MeshViews {
  float P[kMeshViews][12];                    // rows 0..2 of the world -> pixel matrix
  const float* depth[kMeshViews];
  const float* image[kMeshViews];
};

__device__ __forceinline__ long long pack_key(int bx, int by, int bz) {
  return ((long long)(bx + kBias) << 42) | ((long long)(by + kBias) << 21) | (long long)(bz + kBias);
}
__device__ __forceinline__ void unpack_key(long long k, int& bx, int& by, int& bz) {
  bx = (int)(k >> 42) - kBias;
  by = (int)((k >> 21) & 0x1fffff) - kBias;
  bz = (int)(k & 0x1fffff) - kBias;
}

// ---------------------------------------------------------------------------- allocation
// The voxel centres in the cube [p - trunc, p + trunc] have indices ceil((p - trunc)/voxel) ..
// floor((p + trunc)/voxel) per axis; with trunc <= 4 voxel they lie in at most 2 bricks per axis.
// Each point writes 8 keys (repeating its first brick where it spans fewer), or kKeyNone 8 times
// when it is NaN or a brick index leaves [kBrickMin, kBrickMax].
__global__ void __launch_bounds__(256)
mesh_brick_keys_kernel(const float* __restrict__ pts, int n, float voxel, float trunc,
                       long long* __restrict__ keys, unsigned long long* __restrict__ dropped) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo[3], hi[3];
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float p = __ldg(pts + (size_t)i * 3 + a);
    const float fl = ceilf(__fdiv_rn(__fsub_rn(p, trunc), voxel));
    const float fh = floorf(__fdiv_rn(__fadd_rn(p, trunc), voxel));
    // voxel index range of the bricks kBrickMin .. kBrickMax (NaN fails both)
    ok = ok && fl >= 8.f * kBrickMin && fh <= 8.f * kBrickMax + 7.f && fl <= fh;
    lo[a] = ok ? ((int)fl >> 3) : 0;
    hi[a] = ok ? min((int)fh >> 3, lo[a] + 1) : 0;
  }
  long long* out = keys + (size_t)i * 8;
  if (!ok) {
#pragma unroll
    for (int s = 0; s < 8; ++s) out[s] = kKeyNone;
    atomicAdd(dropped, 1ull);
    return;
  }
#pragma unroll
  for (int s = 0; s < 8; ++s)
    out[s] = pack_key(min(lo[0] + (s & 1), hi[0]), min(lo[1] + ((s >> 1) & 1), hi[1]),
                      min(lo[2] + (s >> 2), hi[2]));
}

// nbr[b][o - 1], o = dx + 2 dy + 4 dz in 1..7: index of brick b + (dx, dy, dz), -1 if absent
__global__ void __launch_bounds__(256)
mesh_brick_neighbors_kernel(const long long* __restrict__ keys, int nb, int* __restrict__ nbr) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nb * 7) return;
  const int b = t / 7, o = t - b * 7 + 1;
  int bx, by, bz;
  unpack_key(__ldg(keys + b), bx, by, bz);
  bx += o & 1; by += (o >> 1) & 1; bz += o >> 2;
  int found = -1;
  if (bx <= kBrickMax + 1 && by <= kBrickMax + 1 && bz <= kBrickMax + 1) {
    const long long k = pack_key(bx, by, bz);
    int l = 0, h = nb;                        // first index with keys[idx] >= k
    while (l < h) {
      const int m = (l + h) >> 1;
      if (__ldg(keys + m) < k) l = m + 1; else h = m;
    }
    if (l < nb && __ldg(keys + l) == k) found = l;
  }
  nbr[t] = found;
}

// ---------------------------------------------------------------------------- integration
__global__ void __launch_bounds__(256)
mesh_integrate_kernel(const __grid_constant__ MeshViews V, int nv, const long long* __restrict__ keys,
                      int nb, float voxel, float trunc, int H, int W, float* __restrict__ tsdf,
                      float* __restrict__ weight, float* __restrict__ color) {
  const size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= (size_t)nb * 512) return;
  const int b = (int)(v >> 9), l = (int)(v & 511);
  int bx, by, bz;
  unpack_key(__ldg(keys + b), bx, by, bz);
  const float X = __fmul_rn((float)(bx * 8 + (l & 7)), voxel);
  const float Y = __fmul_rn((float)(by * 8 + ((l >> 3) & 7)), voxel);
  const float Z = __fmul_rn((float)(bz * 8 + (l >> 6)), voxel);
  float s = tsdf[v], w = weight[v];
  float c0 = color[v * 3], c1 = color[v * 3 + 1], c2 = color[v * 3 + 2];
  const float Wf = (float)W, Hf = (float)H;
  for (int k = 0; k < nv; ++k) {
    const float* A = V.P[k];
    // ((A0 X + A1 Y) + A2 Z) + A3 per row
    const float z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A[8], X), __fmul_rn(A[9], Y)),
                                        __fmul_rn(A[10], Z)), A[11]);
    if (!(z > 0.f)) continue;
    const float uz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A[0], X), __fmul_rn(A[1], Y)),
                                         __fmul_rn(A[2], Z)), A[3]);
    const float vz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A[4], X), __fmul_rn(A[5], Y)),
                                         __fmul_rn(A[6], Z)), A[7]);
    const float fx = floorf(__fadd_rn(__fdiv_rn(uz, z), 0.5f));
    const float fy = floorf(__fadd_rn(__fdiv_rn(vz, z), 0.5f));
    if (!(fx >= 0.f && fx < Wf && fy >= 0.f && fy < Hf)) continue;
    const size_t pix = (size_t)(int)fy * W + (int)fx;
    const float D = __ldg(V.depth[k] + pix);
    if (D == 0.f) continue;
    const float sdf = __fsub_rn(D, z);
    if (!(sdf >= -trunc)) continue;
    const float t = fminf(1.f, __fdiv_rn(sdf, trunc));
    const float w1 = __fadd_rn(w, 1.f);
    const float* im = V.image[k] + pix * 3;
    s = __fdiv_rn(__fadd_rn(__fmul_rn(s, w), t), w1);
    c0 = __fdiv_rn(__fadd_rn(__fmul_rn(c0, w), __ldg(im)), w1);
    c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c1, w), __ldg(im + 1)), w1);
    c2 = __fdiv_rn(__fadd_rn(__fmul_rn(c2, w), __ldg(im + 2)), w1);
    w = w1;
  }
  tsdf[v] = s;
  weight[v] = w;
  color[v * 3] = c0; color[v * 3 + 1] = c1; color[v * 3 + 2] = c2;
}

// ---------------------------------------------------------------------------- extraction
// Voxel index of corner c (= dx + 2 dy + 4 dz) of the cell whose lower corner is voxel (b, l),
// -1 when its brick is not allocated.
__device__ __forceinline__ int corner_voxel(const int* __restrict__ nbr, int b, int l, int c) {
  const int x = (l & 7) + (c & 1), y = ((l >> 3) & 7) + ((c >> 1) & 1), z = (l >> 6) + (c >> 2);
  const int o = (x >> 3) | ((y >> 3) << 1) | ((z >> 3) << 2);
  const int bb = o ? __ldg(nbr + (size_t)b * 7 + o - 1) : b;
  return bb < 0 ? -1 : bb * 512 + (((z & 7) * 8 + (y & 7)) * 8 + (x & 7));
}

__device__ __forceinline__ int edge_lower_corner(int e) {
  const int axis = e >> 2, k = e & 3;
  const int o0 = axis == 0 ? 1 : 0, o1 = axis == 2 ? 1 : 2;
  return ((k & 1) << o0) | ((k >> 1) << o1);
}

__global__ void __launch_bounds__(256)
mesh_count_kernel(const int* __restrict__ nbr, int nb, const float* __restrict__ tsdf,
                  const float* __restrict__ weight, unsigned char* __restrict__ cases,
                  int* __restrict__ tri_count, int* __restrict__ edge_used) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nb * 512) return;
  const int b = v >> 9, l = v & 511;
  int cv[8], cs = 0;
  bool valid = true;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    cv[c] = corner_voxel(nbr, b, l, c);
    valid = valid && cv[c] >= 0 && __ldg(weight + cv[c]) > 0.f;
    if (valid && __ldg(tsdf + cv[c]) < 0.f) cs |= 1 << c;
  }
  const int n = valid ? kMcTriCount[cs] : 0;
  cases[v] = (unsigned char)cs;
  tri_count[v] = n;
  if (n == 0) return;
  const unsigned mask = kMcEdgeMask[cs];
  for (int e = 0; e < 12; ++e)                // benign race: every writer stores 1
    if (mask >> e & 1) edge_used[(size_t)cv[edge_lower_corner(e)] * 3 + (e >> 2)] = 1;
}

__global__ void __launch_bounds__(256)
mesh_vertices_kernel(const long long* __restrict__ keys, const int* __restrict__ nbr, int nb,
                     double voxel, const float* __restrict__ tsdf, const float* __restrict__ color,
                     const int* __restrict__ edge_used, const int* __restrict__ edge_scan,
                     float* __restrict__ verts, unsigned char* __restrict__ vcolor) {
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (size_t)nb * 512 * 3 || !__ldg(edge_used + q)) return;
  const int v = (int)(q / 3), axis = (int)(q - (size_t)v * 3);
  const int b = v >> 9, l = v & 511;
  const int u = corner_voxel(nbr, b, l, 1 << axis);
  const double s0 = __ldg(tsdf + v), s1 = __ldg(tsdf + u);
  const double t = __ddiv_rn(s0, __dsub_rn(s0, s1));
  int bi[3];
  unpack_key(__ldg(keys + b), bi[0], bi[1], bi[2]);
  const int li[3] = {l & 7, (l >> 3) & 7, l >> 6};
  const int id = __ldg(edge_scan + q) - 1;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double i = (double)(bi[a] * 8 + li[a]);
    verts[(size_t)id * 3 + a] = (float)__dmul_rn(a == axis ? __dadd_rn(i, t) : i, voxel);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double c0 = __ldg(color + (size_t)v * 3 + c), c1 = __ldg(color + (size_t)u * 3 + c);
    const double x = rint(__dadd_rn(c0, __dmul_rn(t, __dsub_rn(c1, c0))));
    vcolor[(size_t)id * 3 + c] = (unsigned char)fmin(255.0, fmax(0.0, x));
  }
}

__global__ void __launch_bounds__(256)
mesh_faces_kernel(const int* __restrict__ nbr, int nb, const unsigned char* __restrict__ cases,
                  const int* __restrict__ tri_count, const int* __restrict__ tri_scan,
                  const int* __restrict__ edge_scan, int* __restrict__ faces) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nb * 512) return;
  const int n = __ldg(tri_count + v);
  if (n == 0) return;
  const int b = v >> 9, l = v & 511, cs = cases[v];
  const int base = __ldg(tri_scan + v) - n;
  for (int k = 0; k < 3 * n; ++k) {
    const int e = kMcTris[cs][k];
    const int owner = corner_voxel(nbr, b, l, edge_lower_corner(e));
    faces[(size_t)base * 3 + k] = __ldg(edge_scan + (size_t)owner * 3 + (e >> 2)) - 1;
  }
}

inline unsigned blocks_for(size_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_mesh_brick_keys(const float* points, int n, float voxel, float trunc,
                                      long long* keys, unsigned long long* dropped, void* stream) {
  CASMVS_REQUIRE(n >= 0, "mesh_brick_keys: n < 0");
  CASMVS_REQUIRE(voxel > 0.f && trunc >= voxel && trunc <= 4.f * voxel,
                 "mesh_brick_keys: need voxel > 0 and voxel <= trunc <= 4 voxel");
  if (n == 0) return 0;
  CASMVS_REQUIRE(points && keys && dropped, "mesh_brick_keys: null pointer");
  mesh_brick_keys_kernel<<<blocks_for(n), 256, 0, as_stream(stream)>>>(points, n, voxel, trunc,
                                                                        keys, dropped);
  return after_launch("mesh_brick_keys");
}

extern "C" int casmvs_mesh_brick_neighbors(const long long* keys, int nb, int* nbr, void* stream) {
  CASMVS_REQUIRE(nb >= 0 && nb <= kMaxBricks, "mesh_brick_neighbors: 0 <= nb <= %lld", kMaxBricks);
  if (nb == 0) return 0;
  CASMVS_REQUIRE(keys && nbr, "mesh_brick_neighbors: null pointer");
  mesh_brick_neighbors_kernel<<<blocks_for((size_t)nb * 7), 256, 0, as_stream(stream)>>>(keys, nb, nbr);
  return after_launch("mesh_brick_neighbors");
}

extern "C" int casmvs_mesh_integrate(const long long* keys, int nb, float voxel, float trunc,
                                     const float* const* depth, const float* const* image,
                                     const float* proj, int n_views, int H, int W, float* tsdf,
                                     float* weight, float* color, void* stream) {
  CASMVS_REQUIRE(nb >= 0 && nb <= kMaxBricks, "mesh_integrate: 0 <= nb <= %lld", kMaxBricks);
  CASMVS_REQUIRE(n_views >= 0 && H > 0 && W > 0 && (size_t)H * W < (1u << 30),
                 "mesh_integrate: bad dims");
  CASMVS_REQUIRE(voxel > 0.f && trunc > 0.f, "mesh_integrate: voxel and trunc must be > 0");
  if (nb == 0 || n_views == 0) return 0;
  CASMVS_REQUIRE(keys && tsdf && weight && color && depth && image && proj,
                 "mesh_integrate: null pointer");
  for (int k = 0; k < n_views; ++k)
    CASMVS_REQUIRE(depth[k] && image[k], "mesh_integrate: null depth or image of view %d", k);
  const size_t nvox = (size_t)nb * 512;
  for (int k0 = 0; k0 < n_views; k0 += kMeshViews) {
    MeshViews V;
    const int nv = min(kMeshViews, n_views - k0);
    for (int k = 0; k < nv; ++k) {
      for (int r = 0; r < 12; ++r) V.P[k][r] = proj[(size_t)(k0 + k) * 16 + r];
      V.depth[k] = depth[k0 + k];
      V.image[k] = image[k0 + k];
    }
    mesh_integrate_kernel<<<blocks_for(nvox), 256, 0, as_stream(stream)>>>(
        V, nv, keys, nb, voxel, trunc, H, W, tsdf, weight, color);
    const int rc = after_launch("mesh_integrate");
    if (rc) return rc;
  }
  return 0;
}

extern "C" int casmvs_mesh_count(const int* nbr, int nb, const float* tsdf, const float* weight,
                                 unsigned char* cases, int* tri_count, int* edge_used,
                                 void* stream) {
  CASMVS_REQUIRE(nb >= 0 && nb <= kMaxBricks, "mesh_count: 0 <= nb <= %lld", kMaxBricks);
  if (nb == 0) return 0;
  CASMVS_REQUIRE(nbr && tsdf && weight && cases && tri_count && edge_used, "mesh_count: null pointer");
  const size_t nvox = (size_t)nb * 512;
  cudaError_t e = cudaMemsetAsync(edge_used, 0, nvox * 3 * sizeof(int), as_stream(stream));
  CASMVS_REQUIRE(e == cudaSuccess, "mesh_count: memset failed: %s", cudaGetErrorString(e));
  mesh_count_kernel<<<blocks_for(nvox), 256, 0, as_stream(stream)>>>(nbr, nb, tsdf, weight, cases,
                                                                      tri_count, edge_used);
  return after_launch("mesh_count");
}

extern "C" int casmvs_mesh_vertices(const long long* keys, const int* nbr, int nb, float voxel,
                                    const float* tsdf, const float* color, const int* edge_used,
                                    const int* edge_scan, float* verts, unsigned char* vcolor,
                                    void* stream) {
  CASMVS_REQUIRE(nb >= 0 && nb <= kMaxBricks, "mesh_vertices: 0 <= nb <= %lld", kMaxBricks);
  CASMVS_REQUIRE(voxel > 0.f, "mesh_vertices: voxel must be > 0");
  if (nb == 0) return 0;
  CASMVS_REQUIRE(keys && nbr && tsdf && color && edge_used && edge_scan && verts && vcolor,
                 "mesh_vertices: null pointer");
  mesh_vertices_kernel<<<blocks_for((size_t)nb * 512 * 3), 256, 0, as_stream(stream)>>>(
      keys, nbr, nb, (double)voxel, tsdf, color, edge_used, edge_scan, verts, vcolor);
  return after_launch("mesh_vertices");
}

extern "C" int casmvs_mesh_faces(const int* nbr, int nb, const unsigned char* cases,
                                 const int* tri_count, const int* tri_scan, const int* edge_scan,
                                 int* faces, void* stream) {
  CASMVS_REQUIRE(nb >= 0 && nb <= kMaxBricks, "mesh_faces: 0 <= nb <= %lld", kMaxBricks);
  if (nb == 0) return 0;
  CASMVS_REQUIRE(nbr && cases && tri_count && tri_scan && edge_scan && faces,
                 "mesh_faces: null pointer");
  mesh_faces_kernel<<<blocks_for((size_t)nb * 512), 256, 0, as_stream(stream)>>>(
      nbr, nb, cases, tri_count, tri_scan, edge_scan, faces);
  return after_launch("mesh_faces");
}
