// Image resamplers of the scan readers, device side (SURVEY.md 8 f-4): (N,H,W,3) uint8 ->
// (N,OH,OW,3) uint8, byte-identical to the two host libraries the reference resizes with.
//
//  casmvs_resize_u8_pil_fwd     Pillow Image.resize(size, BILINEAR), the network input path
//                               (datasets/{dtu,tanks,blendedmvs}.py img.resize(img_wh, BILINEAR)).
//                               Pillow's 8-bit resampler is separable integer arithmetic: a
//                               horizontal pass into a uint8 intermediate, then a vertical pass,
//                               each  clip8(((1 << 21) + sum_k in[lo + k] * coef[k]) >> 22),  a pass
//                               skipped when its dimension does not change.
//  casmvs_resize_u8_linear_fwd  cv2.resize(INTER_LINEAR) on 8-bit images, the fusion-colour path
//                               (eval.py:266-268): 11-bit weights, an int32 horizontal pass
//                               h = in[x0]*a0 + in[x1]*a1, then the vertical pass of OpenCV's
//                               8-bit specialisation ((b0*(h0>>4))>>16) + ((b1*(h1>>4))>>16),
//                               rounded by (v + 2) >> 2.  Fused: no intermediate.
//
// The host computes the bounds and weight tables once per (input, output) size pair
// (casmvsnet_pl_b200/io.py); the kernels only gather and multiply-accumulate integers.
#include "common.cuh"

namespace casmvs {

// One Pillow pass along W (VERT = false) or H (VERT = true).  One thread per output byte.
// in (N,H,W,3); out (N,H,OW,3) or (N,OH,W,3); bounds (O,2) = (first tap, taps); coef (O,ks).
template <bool VERT>
__global__ void __launch_bounds__(256)
pil_pass_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int N, int H, int W,
                int O, const int* __restrict__ bounds, const int* __restrict__ coef, int ks) {
  const int OH = VERT ? O : H, OW = VERT ? W : O;
  const size_t total = (size_t)N * OH * OW * 3;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % 3);
    const size_t p = i / 3;
    const int ox = (int)(p % OW);
    const size_t q = p / OW;
    const int oy = (int)(q % OH);
    const size_t n = q / OH;
    const int o = VERT ? oy : ox;
    const int lo = __ldg(bounds + 2 * o), taps = __ldg(bounds + 2 * o + 1);
    const int* k = coef + (size_t)o * ks;
    const uint8_t* src = VERT ? in + ((n * H + lo) * W + ox) * 3 + c
                              : in + ((n * H + oy) * W + lo) * 3 + c;
    const size_t step = VERT ? (size_t)W * 3 : 3;
    int acc = 1 << 21;
    for (int t = 0; t < taps; ++t) acc += (int)__ldg(src + t * step) * __ldg(k + t);
    acc >>= 22;
    out[i] = (uint8_t)(acc < 0 ? 0 : acc > 255 ? 255 : acc);
  }
}

// cv2 INTER_LINEAR, both passes.  xtab (OW,4) / ytab (OH,4) = (i0, i1, w0, w1).
__global__ void __launch_bounds__(256)
cv_linear_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int N, int H, int W,
                 int OH, int OW, const int4* __restrict__ xtab, const int4* __restrict__ ytab) {
  const size_t total = (size_t)N * OH * OW * 3;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % 3);
    const size_t p = i / 3;
    const int ox = (int)(p % OW);
    const size_t q = p / OW;
    const int oy = (int)(q % OH);
    const size_t n = q / OH;
    const int4 xt = __ldg(xtab + ox), yt = __ldg(ytab + oy);
    const uint8_t* r0 = in + ((n * H + yt.x) * W) * 3 + c;
    const uint8_t* r1 = in + ((n * H + yt.y) * W) * 3 + c;
    const int h0 = (int)__ldg(r0 + xt.x * 3) * xt.z + (int)__ldg(r0 + xt.y * 3) * xt.w;
    const int h1 = (int)__ldg(r1 + xt.x * 3) * xt.z + (int)__ldg(r1 + xt.y * 3) * xt.w;
    const int v = ((yt.z * (h0 >> 4)) >> 16) + ((yt.w * (h1 >> 4)) >> 16);
    out[i] = (uint8_t)((v + 2) >> 2);
  }
}

inline unsigned grid_for(size_t total) {
  const size_t b = (total + 255) / 256;
  const size_t cap = (size_t)num_sms() * 16;
  return (unsigned)(b < 1 ? 1 : b < cap ? b : cap);
}

}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_resize_u8_pil_fwd(const uint8_t* images, uint8_t* out, uint8_t* tmp, int N,
                                        int H, int W, int OH, int OW, const int* xbounds,
                                        const int* xcoef, int xks, const int* ybounds,
                                        const int* ycoef, int yks, void* stream) {
  CASMVS_REQUIRE(images && out, "resize_u8_pil: null pointer");
  CASMVS_REQUIRE(N >= 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "resize_u8_pil: bad dims");
  const bool horiz = OW != W, vert = OH != H;
  CASMVS_REQUIRE(!horiz || (xbounds && xcoef && xks > 0), "resize_u8_pil: missing x tables");
  CASMVS_REQUIRE(!vert || (ybounds && ycoef && yks > 0), "resize_u8_pil: missing y tables");
  CASMVS_REQUIRE(!(horiz && vert) || tmp, "resize_u8_pil: both passes need tmp (N,H,OW,3)");
  if (N == 0) return 0;
  cudaStream_t st = as_stream(stream);
  if (!horiz && !vert) {
    const cudaError_t e = cudaMemcpyAsync(out, images, (size_t)N * H * W * 3,
                                          cudaMemcpyDeviceToDevice, st);
    CASMVS_REQUIRE(e == cudaSuccess, "resize_u8_pil: copy failed: %s", cudaGetErrorString(e));
    return 0;
  }
  if (horiz) {
    uint8_t* dst = vert ? tmp : out;
    pil_pass_kernel<false><<<grid_for((size_t)N * H * OW * 3), 256, 0, st>>>(
        images, dst, N, H, W, OW, xbounds, xcoef, xks);
    const int rc = after_launch("resize_u8_pil/horizontal");
    if (rc) return rc;
  }
  if (vert) {
    const uint8_t* src = horiz ? tmp : images;
    pil_pass_kernel<true><<<grid_for((size_t)N * OH * OW * 3), 256, 0, st>>>(
        src, out, N, H, OW, OH, ybounds, ycoef, yks);
    return after_launch("resize_u8_pil/vertical");
  }
  return 0;
}

extern "C" int casmvs_resize_u8_linear_fwd(const uint8_t* images, uint8_t* out, int N, int H,
                                           int W, int OH, int OW, const int* xtab,
                                           const int* ytab, void* stream) {
  CASMVS_REQUIRE(images && out && xtab && ytab, "resize_u8_linear: null pointer");
  CASMVS_REQUIRE(N >= 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "resize_u8_linear: bad dims");
  CASMVS_REQUIRE(((reinterpret_cast<uintptr_t>(xtab) | reinterpret_cast<uintptr_t>(ytab)) & 15) == 0,
                 "resize_u8_linear: tables must be 16-byte aligned");
  if (N == 0) return 0;
  cv_linear_kernel<<<grid_for((size_t)N * OH * OW * 3), 256, 0, as_stream(stream)>>>(
      images, out, N, H, W, OH, OW, reinterpret_cast<const int4*>(xtab),
      reinterpret_cast<const int4*>(ytab));
  return after_launch("resize_u8_linear");
}
