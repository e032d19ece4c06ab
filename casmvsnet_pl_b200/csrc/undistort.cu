// Undistortion of distorted COLMAP views, device side: N uint8 RGB images (N,H,W,3) of one
// source camera -> (N,OH,OW,3) in its undistorted PINHOLE camera (casmvsnet_pl_b200/colmap.py
// undistorted_camera).  Per output pixel (x, y), in float64:
//
//   u = (x + 0.5 - cx') / fx',  v = (y + 0.5 - cy') / fy'
//   (du, dv) = COLMAP's forward distortion of the source model,  X = fx (u + du) + cx,  Y likewise
//   sx = X - 0.5, sy = Y - 0.5: 0 in every channel when either lies more than 1e-6 outside
//   [0, W-1] / [0, H-1] (or is not finite), else clamped into it
//   x0 = min(floor(sx), W-2), ax = sx - x0 (y likewise)
//   out = floor((1-ay)((1-ax) p00 + ax p10) + ay((1-ax) p01 + ax p11) + 0.5)
//
// Every operation is an explicitly rounded intrinsic, so nothing is contracted into an FMA and
// oracle/undistort_oracle.py's numpy restatement gives the same bytes for the perspective models.
// The fisheye models call atan, whose last bit may differ from numpy's.
//
// One thread per output pixel computes the map once and applies it to all N images (the
// pipeline passes the Pillow and the cv2 decode of a view together).  Source reads go through
// the read-only path; consecutive threads write consecutive pixels.
#include "common.cuh"

namespace casmvs {

namespace {

enum Model {
  kSimplePinhole = 0, kPinhole = 1, kSimpleRadial = 2, kRadial = 3, kOpenCV = 4,
  kOpenCVFisheye = 5, kFullOpenCV = 6, kSimpleRadialFisheye = 8, kRadialFisheye = 9
};

// The source camera and the undistorted camera, passed by value in the launch.
struct UndistortParams {
  double fx, fy, cx, cy;       // source
  double k[8];                 // distortion coefficients in COLMAP's order, zero-padded
  double ofx, ofy, ocx, ocy;   // undistorted PINHOLE
};

__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dvd(double a, double b) { return __ddiv_rn(a, b); }

// (du, dv) of normalised (u, v); the order of operations is oracle/undistort_oracle.distort's.
template <int M>
__device__ __forceinline__ void distort(const UndistortParams& p, double u, double v, double& du,
                                        double& dv) {
  if (M == kSimplePinhole || M == kPinhole) {
    du = 0.0;
    dv = 0.0;
    return;
  }
  const double u2 = mul(u, u), v2 = mul(v, v), uv = mul(u, v);
  const double r2 = add(u2, v2);
  if (M == kSimpleRadialFisheye || M == kRadialFisheye || M == kOpenCVFisheye) {
    const double r = __dsqrt_rn(r2);
    if (!(r > 0.0)) {
      du = 0.0;
      dv = 0.0;
      return;
    }
    const double th = atan(r);
    const double t2 = mul(th, th);
    double thd;
    if (M == kSimpleRadialFisheye) {
      thd = mul(th, add(1.0, mul(p.k[0], t2)));
    } else if (M == kRadialFisheye) {
      const double t4 = mul(t2, t2);
      thd = mul(th, add(add(1.0, mul(p.k[0], t2)), mul(p.k[1], t4)));
    } else {
      const double t4 = mul(t2, t2);
      const double t6 = mul(t4, t2), t8 = mul(t4, t4);
      thd = mul(th, add(add(add(add(1.0, mul(p.k[0], t2)), mul(p.k[1], t4)), mul(p.k[2], t6)),
                        mul(p.k[3], t8)));
    }
    du = sub(dvd(mul(u, thd), r), u);
    dv = sub(dvd(mul(v, thd), r), v);
    return;
  }
  const double r4 = mul(r2, r2);
  if (M == kSimpleRadial) {
    const double rad = mul(p.k[0], r2);
    du = mul(u, rad);
    dv = mul(v, rad);
    return;
  }
  double rad;
  if (M == kFullOpenCV) {
    const double r6 = mul(r4, r2);
    const double num = add(add(add(1.0, mul(p.k[0], r2)), mul(p.k[1], r4)), mul(p.k[4], r6));
    const double den = add(add(add(1.0, mul(p.k[5], r2)), mul(p.k[6], r4)), mul(p.k[7], r6));
    rad = dvd(num, den);
  } else {
    rad = add(mul(p.k[0], r2), mul(p.k[1], r4));
  }
  if (M == kRadial) {
    du = mul(u, rad);
    dv = mul(v, rad);
    return;
  }
  const double p1 = p.k[2], p2 = p.k[3];
  du = add(add(mul(u, rad), mul(mul(2.0, p1), uv)), mul(p2, add(r2, mul(2.0, u2))));
  dv = add(add(mul(v, rad), mul(mul(2.0, p2), uv)), mul(p1, add(r2, mul(2.0, v2))));
  if (M == kFullOpenCV) {
    du = sub(du, u);
    dv = sub(dv, v);
  }
}

template <int M>
__global__ void __launch_bounds__(256)
undistort_u8_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int N, int H,
                    int W, int OH, int OW, const UndistortParams p) {
  const size_t npix = (size_t)OH * OW;
  const size_t in_plane = (size_t)H * W * 3, out_plane = npix * 3;
  const double xmax = add((double)(W - 1), 1e-6), ymax = add((double)(H - 1), 1e-6);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix;
       i += (size_t)gridDim.x * blockDim.x) {
    const int ox = (int)(i % OW), oy = (int)(i / OW);
    const double u = dvd(sub(add((double)ox, 0.5), p.ocx), p.ofx);
    const double v = dvd(sub(add((double)oy, 0.5), p.ocy), p.ofy);
    double du, dv;
    distort<M>(p, u, v, du, dv);
    double sx = sub(add(mul(p.fx, add(u, du)), p.cx), 0.5);
    double sy = sub(add(mul(p.fy, add(v, dv)), p.cy), 0.5);
    uint8_t* o = out + i * 3;
    if (!(sx >= -1e-6 && sx <= xmax && sy >= -1e-6 && sy <= ymax)) {   // NaN and inf fail too
      for (int n = 0; n < N; ++n, o += out_plane) o[0] = o[1] = o[2] = 0;
      continue;
    }
    sx = fmin(fmax(sx, 0.0), (double)(W - 1));
    sy = fmin(fmax(sy, 0.0), (double)(H - 1));
    const int x0 = min((int)floor(sx), W - 2), y0 = min((int)floor(sy), H - 2);
    const double ax = sub(sx, (double)x0), ay = sub(sy, (double)y0);
    const double bx = sub(1.0, ax), by = sub(1.0, ay);
    const uint8_t* s = in + ((size_t)y0 * W + x0) * 3;
    const size_t row = (size_t)W * 3;
    for (int n = 0; n < N; ++n, s += in_plane, o += out_plane) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double p00 = __ldg(s + c), p10 = __ldg(s + 3 + c);
        const double p01 = __ldg(s + row + c), p11 = __ldg(s + row + 3 + c);
        const double val = add(mul(by, add(mul(bx, p00), mul(ax, p10))),
                               mul(ay, add(mul(bx, p01), mul(ax, p11))));
        const double r = floor(add(val, 0.5));
        o[c] = (uint8_t)(r < 0.0 ? 0.0 : r > 255.0 ? 255.0 : r);
      }
    }
  }
}

unsigned grid_for_pixels(size_t npix) {
  const size_t b = (npix + 255) / 256;
  const size_t cap = (size_t)num_sms() * 16;
  return (unsigned)(b < 1 ? 1 : b < cap ? b : cap);
}

}  // namespace

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_undistort_u8_fwd(const uint8_t* images, uint8_t* out, int N, int H, int W,
                                       int OH, int OW, int model, const double* src_params,
                                       const double* dst_params, void* stream) {
  int n_params = 0;
  switch (model) {
    case kSimplePinhole: n_params = 3; break;
    case kPinhole: n_params = 4; break;
    case kSimpleRadial: case kSimpleRadialFisheye: n_params = 4; break;
    case kRadial: case kRadialFisheye: n_params = 5; break;
    case kOpenCV: case kOpenCVFisheye: n_params = 8; break;
    case kFullOpenCV: n_params = 12; break;
    default: CASMVS_REQUIRE(false, "undistort_u8: unsupported camera model id %d", model);
  }
  CASMVS_REQUIRE(N >= 0 && H >= 2 && W >= 2 && OH > 0 && OW > 0,
                 "undistort_u8: bad dims N=%d H=%d W=%d OH=%d OW=%d (the source needs 2x2)", N, H,
                 W, OH, OW);
  CASMVS_REQUIRE(src_params && dst_params, "undistort_u8: null parameter array");
  CASMVS_REQUIRE(N == 0 || (images && out), "undistort_u8: null pointer");
  UndistortParams p{};
  const bool single = model == kSimplePinhole || model == kSimpleRadial || model == kRadial ||
                      model == kSimpleRadialFisheye || model == kRadialFisheye;
  const int nf = single ? 3 : 4;                  // f, cx, cy  or  fx, fy, cx, cy
  p.fx = src_params[0];
  p.fy = single ? src_params[0] : src_params[1];
  p.cx = src_params[nf - 2];
  p.cy = src_params[nf - 1];
  for (int j = nf; j < n_params; ++j) p.k[j - nf] = src_params[j];
  p.ofx = dst_params[0];
  p.ofy = dst_params[1];
  p.ocx = dst_params[2];
  p.ocy = dst_params[3];
  CASMVS_REQUIRE(p.fx > 0 && p.fy > 0 && p.ofx > 0 && p.ofy > 0,
                 "undistort_u8: focal lengths must be positive");
  if (N == 0) return 0;
  const unsigned grid = grid_for_pixels((size_t)OH * OW);
  cudaStream_t st = as_stream(stream);
#define CASMVS_UNDISTORT_CASE(M)                                                               \
  case M:                                                                                      \
    undistort_u8_kernel<M><<<grid, 256, 0, st>>>(images, out, N, H, W, OH, OW, p);             \
    break;
  switch (model) {
    CASMVS_UNDISTORT_CASE(kSimplePinhole)
    CASMVS_UNDISTORT_CASE(kPinhole)
    CASMVS_UNDISTORT_CASE(kSimpleRadial)
    CASMVS_UNDISTORT_CASE(kRadial)
    CASMVS_UNDISTORT_CASE(kOpenCV)
    CASMVS_UNDISTORT_CASE(kOpenCVFisheye)
    CASMVS_UNDISTORT_CASE(kFullOpenCV)
    CASMVS_UNDISTORT_CASE(kSimpleRadialFisheye)
    CASMVS_UNDISTORT_CASE(kRadialFisheye)
  }
#undef CASMVS_UNDISTORT_CASE
  return after_launch("undistort_u8");
}
