// K2 (fp32 CUDA-core variant) — 3x3x3 convolution / transposed convolution on
// channels-last volumes with the norm-act (+skip) epilogue fused.
//
// Replaces (reference, relative to /root/reference):
//   ConvBnReLU3D                       models/modules.py:21-31
//   ConvTranspose3d + norm_act         models/mvsnet.py:74-87
//   skip additions, prob head          models/mvsnet.py:91-104
//
// This is the bit-faithful-products path (CASMVS_FP32: every layer of both networks, the
// data gradients of the training path) and the counted fallback of the TF32 mode for a layer
// shape no tensor-core kernel covers (casmvs_fallback_count; none in the reference architecture).
//
// Thread = TW consecutive-w output voxels x COT output channels.  The block's
// slice of the packed weights ([27][Cin][COT]) sits in shared memory and is read
// with warp-broadcast LDS.128; activations are float4 (4 input channels) loads.
#include "common.cuh"

namespace casmvs {

enum { K_CONV_S1 = 0, K_CONV_S2 = 1, K_CONVT = 2 };
constexpr int kConvThreads = 128;

struct ConvDims {
  int B, Cin, Cout;
  int Di, hi, wi;  // input
  int Do, ho, wo;  // output
  int kd_lo, kd_hi;  // depth taps to visit: [0,3) for a 3x3x3 kernel, [1,2) for a planar (1x3x3) one
};

template <int COT>
__device__ __forceinline__ void load_w(const float* __restrict__ s, float (&wv)[COT]) {
  if constexpr (COT == 8) {
    float4 a = *reinterpret_cast<const float4*>(s), b = *reinterpret_cast<const float4*>(s + 4);
    wv[0] = a.x; wv[1] = a.y; wv[2] = a.z; wv[3] = a.w;
    wv[4] = b.x; wv[5] = b.y; wv[6] = b.z; wv[7] = b.w;
  } else {
#pragma unroll
    for (int k = 0; k < COT; ++k) wv[k] = s[k];
  }
}

template <int KIND, int TW, int COT>
__global__ void __launch_bounds__(kConvThreads)
conv3d_direct_kernel(const float* __restrict__ x, const float* __restrict__ wpk,
                     const float* __restrict__ scale, const float* __restrict__ shift,
                     float slope, const float* __restrict__ skip, float* __restrict__ y,
                     ConvDims dm, int round_out) {
  extern __shared__ __align__(16) float s_w[];  // [27][Cin][COT]
  const int Cin = dm.Cin, Cout = dm.Cout;
  const int co0 = blockIdx.y * COT;
  for (int i = threadIdx.x; i < 27 * Cin * COT; i += blockDim.x) {
    int k = i % COT, r = i / COT;                // r = tap*Cin + ci
    s_w[i] = (co0 + k < Cout) ? wpk[(size_t)r * Cout + co0 + k] : 0.f;
  }
  __syncthreads();

  const int wgroups = (dm.wo + TW - 1) / TW;
  const long total = (long)dm.B * dm.Do * dm.ho * wgroups;
  const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int wg = (int)(gid % wgroups);
  long t = gid / wgroups;
  const int oh = (int)(t % dm.ho); t /= dm.ho;
  const int od = (int)(t % dm.Do);
  const int b = (int)(t / dm.Do);
  const int ow0 = wg * TW;

  float acc[TW][COT];
#pragma unroll
  for (int j = 0; j < TW; ++j)
#pragma unroll
    for (int k = 0; k < COT; ++k) acc[j][k] = 0.f;

  const float* xb = x + (size_t)b * dm.Di * dm.hi * dm.wi * Cin;

  if constexpr (KIND == K_CONV_S1) {
    for (int kd = dm.kd_lo; kd < dm.kd_hi; ++kd) {
      const int id = od + kd - 1;
      if (id < 0 || id >= dm.Di) continue;
      for (int kh = 0; kh < 3; ++kh) {
        const int ih = oh + kh - 1;
        if (ih < 0 || ih >= dm.hi) continue;
        const float* row = xb + ((size_t)id * dm.hi + ih) * dm.wi * Cin;
        const float* wrow = s_w + (size_t)((kd * 3 + kh) * 3) * Cin * COT;
        for (int ci = 0; ci < Cin; ci += 4) {
          float4 in[TW + 2];
#pragma unroll
          for (int j = 0; j < TW + 2; ++j) {
            const int iw = ow0 + j - 1;
            in[j] = (iw >= 0 && iw < dm.wi) ? ldg4(row + (size_t)iw * Cin + ci)
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) {
              float wv[COT];
              load_w<COT>(wrow + ((size_t)kw * Cin + ci + cc) * COT, wv);
#pragma unroll
              for (int j = 0; j < TW; ++j) {
                const float4 v4 = in[j + kw];
                const float v = cc == 0 ? v4.x : cc == 1 ? v4.y : cc == 2 ? v4.z : v4.w;
#pragma unroll
                for (int k = 0; k < COT; ++k) acc[j][k] = fmaf(v, wv[k], acc[j][k]);
              }
            }
          }
        }
      }
    }
  } else {
    // generic gather: TW == 1.  conv stride 2: i = 2*o + k - 1.
    // transposed (s2,p1,op1): o = 2*i - 1 + k  =>  i = (o + 1 - k)/2 when even.
    static_assert(KIND == K_CONV_S1 || TW == 1, "strided kinds use TW=1");
    for (int kd = 0; kd < 3; ++kd) {
      int id;
      if (KIND == K_CONV_S2) { id = 2 * od + kd - 1; }
      else { int n = od + 1 - kd; if (n < 0 || (n & 1)) continue; id = n >> 1; }
      if (id < 0 || id >= dm.Di) continue;
      for (int kh = 0; kh < 3; ++kh) {
        int ih;
        if (KIND == K_CONV_S2) { ih = 2 * oh + kh - 1; }
        else { int n = oh + 1 - kh; if (n < 0 || (n & 1)) continue; ih = n >> 1; }
        if (ih < 0 || ih >= dm.hi) continue;
        for (int kw = 0; kw < 3; ++kw) {
          int iw;
          if (KIND == K_CONV_S2) { iw = 2 * ow0 + kw - 1; }
          else { int n = ow0 + 1 - kw; if (n < 0 || (n & 1)) continue; iw = n >> 1; }
          if (iw < 0 || iw >= dm.wi) continue;
          const float* px = xb + (((size_t)id * dm.hi + ih) * dm.wi + iw) * Cin;
          const float* wrow = s_w + (size_t)((kd * 3 + kh) * 3 + kw) * Cin * COT;
          for (int ci = 0; ci < Cin; ci += 4) {
            const float4 v4 = ldg4(px + ci);
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) {
              float wv[COT];
              load_w<COT>(wrow + (size_t)(ci + cc) * COT, wv);
              const float v = cc == 0 ? v4.x : cc == 1 ? v4.y : cc == 2 ? v4.z : v4.w;
#pragma unroll
              for (int k = 0; k < COT; ++k) acc[0][k] = fmaf(v, wv[k], acc[0][k]);
            }
          }
        }
      }
    }
  }

  // epilogue: y = act(acc*scale + shift) + skip      (ABN eval: x*alpha + beta, LeakyReLU)
  float sc[COT], sh[COT];
#pragma unroll
  for (int k = 0; k < COT; ++k) {
    const bool ok = co0 + k < Cout;
    sc[k] = ok ? (scale ? __ldg(scale + co0 + k) : 1.f) : 0.f;
    sh[k] = ok ? (shift ? __ldg(shift + co0 + k) : 0.f) : 0.f;
  }
#pragma unroll
  for (int j = 0; j < TW; ++j) {
    const int ow = ow0 + j;
    if (ow >= dm.wo) break;
    const size_t o = ((((size_t)b * dm.Do + od) * dm.ho + oh) * dm.wo + ow) * Cout + co0;
    float v[COT];
#pragma unroll
    for (int k = 0; k < COT; ++k) {
      float t2 = fmaf(acc[j][k], sc[k], sh[k]);
      v[k] = t2 >= 0.f ? t2 : t2 * slope;
    }
    if constexpr (COT == 8) {
      if (skip) {
        float4 s0 = ldg4(skip + o), s1 = ldg4(skip + o + 4);
        v[0] += s0.x; v[1] += s0.y; v[2] += s0.z; v[3] += s0.w;
        v[4] += s1.x; v[5] += s1.y; v[6] += s1.z; v[7] += s1.w;
      }
      if (round_out) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          uint32_t r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v[k])); v[k] = __uint_as_float(r);
        }
      }
      st4(y + o, make_float4(v[0], v[1], v[2], v[3]));
      st4(y + o + 4, make_float4(v[4], v[5], v[6], v[7]));
    } else {
#pragma unroll
      for (int k = 0; k < COT; ++k)
        if (co0 + k < Cout) y[o + k] = v[k] + (skip ? __ldg(skip + o + k) : 0.f);
    }
  }
}

// (Cout,Cin,27) [Conv3d] or (Cin,Cout,27) [ConvTranspose3d] -> [27][Cin][Cout].
// For the transposed conv the tap index is kept as torch's k (o = 2i - 1 + k).
__global__ void pack_w_kernel(const float* __restrict__ wt, float* __restrict__ wp, int kind,
                              int Cin, int Cout) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = 27 * Cin * Cout;
  if (i >= n) return;
  const int co = i % Cout;
  const int ci = (i / Cout) % Cin;
  const int tap = i / (Cout * Cin);
  if (kind == CASMVS_CONV_PLANAR) {        // (Cout,Cin,3,3) -> centre plane, outer planes zero
    wp[i] = (tap >= 9 && tap < 18) ? wt[((size_t)co * Cin + ci) * 9 + (tap - 9)] : 0.f;
    return;
  }
  const size_t src = kind == CASMVS_CONV ? ((size_t)co * Cin + ci) * 27 + tap
                                         : ((size_t)ci * Cout + co) * 27 + tap;
  wp[i] = wt[src];
}

template <int KIND, int TW>
static int launch_direct(const float* x, const float* wpk, const float* scale, const float* shift,
                         float slope, const float* skip, float* y, const ConvDims& dm,
                         cudaStream_t st, int round_out) {
  const int wgroups = (dm.wo + TW - 1) / TW;
  const long total = (long)dm.B * dm.Do * dm.ho * wgroups;
  if (total == 0) return 0;
  const long blocks = (total + kConvThreads - 1) / kConvThreads;
  CASMVS_REQUIRE(blocks < (1l << 31), "conv3d: volume too large");
  if (dm.Cout % 8 == 0) {
    const size_t smem = (size_t)27 * dm.Cin * 8 * sizeof(float);
    auto kfn = conv3d_direct_kernel<KIND, TW, 8>;
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kfn<<<dim3((unsigned)blocks, dm.Cout / 8), kConvThreads, smem, st>>>(x, wpk, scale, shift,
                                                                       slope, skip, y, dm, round_out);
  } else {
    CASMVS_REQUIRE(dm.Cout == 1, "conv3d: Cout must be 1 or a multiple of 8 (got %d)", dm.Cout);
    const size_t smem = (size_t)27 * dm.Cin * sizeof(float);
    conv3d_direct_kernel<KIND, TW, 1><<<dim3((unsigned)blocks, 1), kConvThreads, smem, st>>>(
        x, wpk, scale, shift, slope, skip, y, dm, 0);
  }
  return after_launch("conv3d_direct");
}

int conv3d_direct(const float* x, const float* wpk, const float* scale, const float* shift,
                  float slope, const float* skip, float* y, int B, int Cin, int Cout, int D,
                  int h, int w, int kind, int stride, cudaStream_t st, int round_out) {
  ConvDims dm;
  dm.B = B; dm.Cin = Cin; dm.Cout = Cout; dm.Di = D; dm.hi = h; dm.wi = w;
  dm.kd_lo = 0; dm.kd_hi = 3;
  if (kind == CASMVS_CONV_PLANAR) {      // the two outer weight planes are zero: skip them
    dm.kd_lo = 1; dm.kd_hi = 2;
    kind = CASMVS_CONV;
  }
  if (kind == CASMVS_CONV) {
    dm.Do = (D - 1) / stride + 1; dm.ho = (h - 1) / stride + 1; dm.wo = (w - 1) / stride + 1;
    if (stride == 1) {
      // small (deep) volumes: one voxel per thread so that the grid still covers the SMs
      const long groups4 = (long)B * dm.Do * dm.ho * ((dm.wo + 3) / 4) * ((Cout + 7) / 8);
      if (groups4 < (long)num_sms() * kConvThreads * 2)
        return launch_direct<K_CONV_S1, 1>(x, wpk, scale, shift, slope, skip, y, dm, st, round_out);
      return launch_direct<K_CONV_S1, 4>(x, wpk, scale, shift, slope, skip, y, dm, st, round_out);
    }
    return launch_direct<K_CONV_S2, 1>(x, wpk, scale, shift, slope, skip, y, dm, st, round_out);
  }
  dm.Do = 2 * D; dm.ho = 2 * h; dm.wo = 2 * w;
  return launch_direct<K_CONVT, 1>(x, wpk, scale, shift, slope, skip, y, dm, st, round_out);
}

}  // namespace casmvs

using namespace casmvs;

extern "C" size_t casmvs_packed_conv3d_weight_floats(int Cin, int Cout) {
  return (size_t)27 * Cin * Cout;
}

extern "C" int casmvs_pack_conv3d_weights(const float* w_torch, int kind, int Cin, int Cout,
                                          float* w_packed, void* stream) {
  CASMVS_REQUIRE(w_torch && w_packed, "pack_conv3d_weights: null pointer");
  CASMVS_REQUIRE(kind == CASMVS_CONV || kind == CASMVS_CONV_TRANSPOSE ||
                     kind == CASMVS_CONV_PLANAR, "pack: bad kind");
  CASMVS_REQUIRE(Cin > 0 && Cout > 0, "pack: bad dims");
  const int n = 27 * Cin * Cout;
  pack_w_kernel<<<(n + 255) / 256, 256, 0, as_stream(stream)>>>(w_torch, w_packed, kind, Cin, Cout);
  return after_launch("pack_conv3d_weights");
}
