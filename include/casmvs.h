/*
 * casmvs.h — C ABI of libcasmvs.so, the H100 (sm_90a) cascade-MVS depth engine.
 *
 * The reference (kwea123/CasMVSNet_pl) has NO FFI layer: its boundary for the
 * hot path is the Python surface models/mvsnet.py + models/modules.py
 * (SURVEY.md §8b).  This header is the C boundary a binding for that surface
 * needs; each entry cites the reference code it replaces (paths relative to
 * the reference root).  The Python binding that mirrors the reference API on
 * top of it lives in casmvsnet_pl_b200/models/ and is shown in INTEGRATION.md.
 *
 * Conventions
 *  - every function returns 0 on success, <0 on error; casmvs_last_error()
 *    returns a thread-local description.  No exceptions cross the boundary.
 *  - all tensor arguments are raw DEVICE pointers owned by the caller (e.g.
 *    torch.Tensor.data_ptr()); the library never allocates or frees
 *    user-visible memory.  Scratch memory is passed in as workspace.
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued on it and
 *    the call returns without synchronising (CUDA-graph capturable).
 *  - fp32 everywhere (the reference declares AMP unsupported, opt.py:69-70);
 *    depth_index is int64 like torch's .long().
 *  - there is no CPU fallback: casmvs_device_check() fails on anything other than
 *    compute capability 9.0 (sm_90a).
 *
 * Memory layouts (enum casmvs_layout)
 *   CASMVS_NCHW : channels-first, the reference's public layout
 *                 features (B,V,C,h,w), volumes (B,C,D,h,w)
 *   CASMVS_NHWC : channels-last, the engine's internal layout
 *                 features (B,V,h,w,C), volumes (B,D,h,w,C)
 */
#ifndef CASMVS_H_
#define CASMVS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CASMVS_VERSION 100  /* 0.1.0 */

enum casmvs_layout { CASMVS_NCHW = 0, CASMVS_NHWC = 1 };
/* OR-ed into casmvs_warp_cost_fwd's cost_layout: store the cost volume rounded to
 * TF32 (round-to-nearest) because the consumer is the wgmma tf32 conv, which
 * would otherwise truncate the operand (biased). */
#define CASMVS_ROUND_TF32 256

/* precision of the 3D-conv contraction (K2) */
enum casmvs_precision {
  CASMVS_FP32 = 0,  /* CUDA-core fp32 FMA (bit-faithful products)            */
  CASMVS_TF32 = 1   /* wgmma tf32, fp32 accumulate in registers         */
};

/* OR-ed into casmvs_conv3d_fwd's precision: store the output unrounded even in the TF32
 * mode (by default activations are stored TF32-rounded there because the next tensor-core
 * layer would otherwise truncate them; the last layer before a non-tensor consumer should
 * keep the fp32 accumulator). */
#define CASMVS_KEEP_FP32_OUT 256

/* Blocked volume layout (B, C/4, D, h, w, 4): channel quads outermost, so one quad of a row of
 * voxels is contiguous.  The CostRegNet driver stores its TF32-mode activations this way.
 * OR-ed into casmvs_costreg_fwd's precision: x is blocked instead of channels-last (where
 * casmvs_costreg_blocked_supported).
 * OR-ed into casmvs_warp_cost_ladder_fwd's round_tf32: write the cost volume blocked. */
#define CASMVS_BLOCKED 512

enum casmvs_conv_kind {
  CASMVS_CONV = 0,           /* Conv3d(k=3, pad=1, stride 1|2)   modules.py:26      */
  CASMVS_CONV_TRANSPOSE = 1, /* ConvTranspose3d(k=3,s=2,p=1,op=1) mvsnet.py:75,80,85 */
  /* 1x3x3 kernel, stride 1, pad (0,1,1): the 3x3 Conv2d layers of FeatureNet
   * (ConvBnReLU modules.py:8-18, smooth0/1 mvsnet.py:30-31) run as ONE convolution over
   * the (views, H, W) volume of a batch.  Packed weights keep the [27][Cin][Cout] layout
   * with zero kd = 0 and kd = 2 planes, so every K2 kernel computes it correctly and the
   * tensor-core kernels skip the two empty planes. */
  CASMVS_CONV_PLANAR = 2
};

/* ---- library / device ------------------------------------------------- */
int casmvs_version(void);
const char* casmvs_last_error(void);
/* 0 iff `device` exists and has compute capability 9.0 (no fallback). */
int casmvs_device_check(int device);
/* number of kernels this library has launched since load (bench evidence). */
uint64_t casmvs_launch_count(void);
/* number of CASMVS_TF32 layers that no wgmma kernel covered and that therefore ran on the
 * CUDA-core kernel (same results up to TF32 rounding, several times slower).  0 for the
 * reference architecture at every BASELINE configuration; bench.py and the full-size tests
 * assert that. */
uint64_t casmvs_fallback_count(void);

/* ---- K1: fused homography warp + bilinear sample + cost reduction ------
 * Replaces homo_warp (models/modules.py:52-92) called V-1 times plus the
 * variance (models/mvsnet.py:137-141,147-156,166-168) or group-wise
 * correlation (:143-144,158-162,170-172) accumulation.  The warped
 * (B,V-1,C,D,h,w) volumes are never materialised.
 *   feats        (B,V,C,h,w) [NCHW] or (B,V,h,w,C) [NHWC]; view 0 = reference
 *   proj         (B,V-1,3,4) row-major  src_proj @ ref_proj^-1
 *   depth_values (B,D,h,w)
 *   cost         num_groups==1: C channels  (B,C,D,h,w)|(B,D,h,w,C)
 *                num_groups >1: G channels  (B,G,D,h,w)|(B,D,h,w,G)
 * Workspace: casmvs_warp_cost_workspace_bytes() (only needed when feats are
 * NCHW: they are re-laid-out once to NHWC).  C % 8 == 0, C % G == 0.
 */
size_t casmvs_warp_cost_workspace_bytes(int feat_layout, int B, int V, int C, int h, int w);
int casmvs_warp_cost_fwd(const float* feats, int feat_layout, const float* proj,
                         const float* depth_values, float* cost, int cost_layout,
                         int B, int V, int C, int D, int h, int w, int num_groups,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Stand-alone homo_warp (models/modules.py:52-92): materialises the warped
 * volume for API completeness.  src_feat (B,C,h,w)|(B,h,w,C), proj (B,3,4),
 * depth_values (B,D,h,w) -> warped (B,C,D,h,w)|(B,D,h,w,C).               */
int casmvs_homo_warp_fwd(const float* src_feat, int feat_layout, const float* proj,
                         const float* depth_values, float* warped, int out_layout,
                         int B, int C, int D, int h, int w, void* stream);

/* ---- K2: 3x3x3 convolution with fused norm-act epilogue ----------------
 * Replaces ConvBnReLU3D (models/modules.py:21-31), the ConvTranspose3d +
 * norm_act pairs and the skip additions of CostRegNet.forward
 * (models/mvsnet.py:60-104) and its `prob` head (:89,103).
 *   y = act( conv(x, w) * scale[c] + shift[c] ) + skip
 *   act(v) = v >= 0 ? v : slope * v   (slope = 1 -> identity, used by `prob`)
 * Volumes are channels-last (B,D,h,w,C).  Weights are pre-packed with
 * casmvs_pack_conv3d_weights (tap-major [27][Cin][Cout]).
 * For kind == CASMVS_CONV: stride in {1,2}, out dims = (in-1)/stride+1.
 * For kind == CASMVS_CONV_TRANSPOSE: out dims = 2*in.
 * For kind == CASMVS_CONV_PLANAR: stride 1, out dims = in dims.
 */
size_t casmvs_packed_conv3d_weight_floats(int Cin, int Cout);
/* w_torch: Conv3d layout (Cout,Cin,3,3,3), ConvTranspose3d layout (Cin,Cout,3,3,3) or, for
 * CASMVS_CONV_PLANAR, Conv2d layout (Cout,Cin,3,3) */
int casmvs_pack_conv3d_weights(const float* w_torch, int kind, int Cin, int Cout,
                               float* w_packed, void* stream);
/* The tensor-core kernels keep a per-process cache of operand images keyed by the w_packed
 * pointer (thread-safe).  An image lives as long as the packed buffer it was built from:
 *   casmvs_release_weight_images(p, bytes) drops the images whose key lies in [p, p+bytes);
 *     call it when a packed buffer is (re)created at an address, rewritten in place or freed
 *     (frees device memory => synchronises with kernels still reading those images);
 *   casmvs_invalidate_weight_cache() drops everything;
 *   casmvs_weight_cache_generation() increases whenever at least one image was dropped: a
 *     captured CUDA graph embeds image pointers and must be re-captured when it changes. */
int casmvs_release_weight_images(const void* w_packed, size_t bytes);
int casmvs_invalidate_weight_cache(void);
uint64_t casmvs_weight_cache_generation(void);
/* number of cached images keyed inside [w_packed, w_packed + bytes): a captured graph records
 * it per packed buffer it depends on and re-checks it before every replay (a release anywhere
 * else -- another model, a dead model's recycled address -- does not invalidate the graph). */
int casmvs_weight_image_count(const void* w_packed, size_t bytes);
/* Synchronises the device and marks every cached image as built.  Call it between the warm-up
 * forward and a CUDA-graph capture: during a capture the cache cannot query or wait on the
 * builders' events (such calls invalidate the capture), so it must already know. */
int casmvs_settle_weight_images(void);
int casmvs_conv3d_fwd(const float* x, const float* w_packed, const float* scale,
                      const float* shift, float slope, const float* skip, float* y,
                      int B, int Cin, int Cout, int D, int h, int w, /* INPUT dims */
                      int kind, int stride, int precision, void* stream);

/* Whole CostRegNet (models/mvsnet.py:91-104) in one call.  `params` is a
 * device array produced by casmvs_costreg_pack (see casmvs_costreg_param_floats).
 * x (B,D,h,w,Cin) -> logits (B,D,h,w) ; D,h,w divisible by 8.
 * precision | CASMVS_BLOCKED: x is (B,Cin/4,D,h,w,4) instead, e.g. the cost volume of
 * casmvs_warp_cost_ladder_fwd with CASMVS_BLOCKED; only where
 * casmvs_costreg_blocked_supported(Cin, precision), an error otherwise.  There the activations
 * in the workspace are blocked as well; the workspace size does not depend on it.          */
size_t casmvs_costreg_param_floats(int Cin);
/* Layout of the params blob: layers 0..10 = conv0..conv6, conv7, conv9, conv11,
 * prob; each is packed weights [27][cin][cout], scale[cout], shift[cout]
 * (scale/shift = folded eval-mode ABN: alpha = gamma/sqrt(var+eps),
 * beta' = beta - mean*alpha; prob: scale = 1, shift = bias).  Offsets in floats. */
int casmvs_costreg_layer_info(int Cin, int layer, int* cin, int* cout, int* kind, int* stride,
                              size_t* w_off, size_t* scale_off, size_t* shift_off);
size_t casmvs_costreg_workspace_bytes(int B, int Cin, int D, int h, int w);
/* 1 when casmvs_costreg_fwd stores its activations blocked for this Cin and precision and so
 * accepts a CASMVS_BLOCKED input (TF32, Cin in {8,16,32}, tensor-core kernels not switched off
 * by CASMVS_TMA / CASMVS_TMA2; x and workspace must then be 16-byte aligned), else 0.  The
 * other cases run channels-last, layers no tensor-core kernel covers on the CUDA cores. */
int casmvs_costreg_blocked_supported(int Cin, int precision);
int casmvs_costreg_fwd(const float* x, const float* params, float* logits,
                       int B, int Cin, int D, int h, int w, int precision,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ---- K3: softmax over D + depth regression + index + confidence --------
 * Replaces F.softmax + depth_regression (models/mvsnet.py:174-177,
 * models/modules.py:95-104) and the confidence block (:179-193).
 *   logits (B,D,h,w); depth_values (B,D,h,w) or, if dv_is_vector, (D,)
 *   depth (B,h,w) f32, confidence (B,h,w) f32,
 *   index (B,h,w) int64 or NULL, prob (B,D,h,w) or NULL.
 * input_is_prob != 0 skips the softmax (logits already hold probabilities).
 * Sums over D use the main-path order of ATen's CPU sum (sequential 16-term
 * chunks, cascaded); depth_index equals the oracle's for identical p.      */
int casmvs_regress_fwd(const float* logits, const float* depth_values, int dv_is_vector,
                       int input_is_prob, float* depth, float* confidence,
                       int64_t* index, float* prob, int B, int D, int h, int w,
                       void* stream);

/* ---- K4: depth hypotheses ----------------------------------------------
 * casmvs_depth_hypotheses_fwd replaces get_depth_values
 * (models/modules.py:34-49): out[b,d] = max(cur - half_range, 1e-7) + step*d.
 * If upsample != 0 `cur` is (B,h/2,w/2) and is first upsampled x2 bilinear,
 * align_corners=True (models/mvsnet.py:231-234); else `cur` is (B,h,w).
 * step_dev (B floats, device) overrides `step`/`half_range` when non-NULL
 * (tensor-valued depth_interval): half_range = fl32(D/2)*step_dev[b].
 * casmvs_uniform_hypotheses_fwd replaces models/mvsnet.py:213-229:
 * out[b,d,:,:] = depth_min + step*d, depth_min/step scalars or device (B,).  */
int casmvs_depth_hypotheses_fwd(const float* cur, int upsample, float half_range,
                                float step, const float* step_dev, float* out,
                                int B, int D, int h, int w, void* stream);
int casmvs_uniform_hypotheses_fwd(float depth_min, float step, const float* depth_min_dev,
                                  const float* step_dev, float* out,
                                  int B, int D, int h, int w, void* stream);

/* ---- cascade-internal forms: hypotheses as a ladder, never materialised -----------------
 * Inside the cascade every pixel's hypotheses are first + step*d (get_depth_values,
 * models/modules.py:44-48; initial planes, models/mvsnet.py:215-229).  These entries take the
 * ladder instead of the (B,D,h,w) tensor and generate it in the kernel with the same two
 * roundings, so K4's D*h*w floats are neither written nor read back by K1 and K3 (bit-identical
 * results).  first: `first_map` (B,h,w) per pixel, else `first_b` (B) per batch item, else the
 * scalar `first`; step: `step_b` (B) else the scalar `step`.
 * casmvs_depth_first_fwd writes only the first rung (B,h,w) of casmvs_depth_hypotheses_fwd.
 * casmvs_warp_cost_ladder_fwd: channels-last features and cost volume; shapes of the staged
 * kernel only (V-1 in {1,2}, C in {8,16,32}, num_groups 1 or 8), error otherwise.
 * round_tf32: nonzero = store the cost TF32-rounded; | CASMVS_BLOCKED = store it blocked,
 * (B,Cout/4,D,h,w,4), for casmvs_costreg_fwd with CASMVS_BLOCKED. */
int casmvs_depth_first_fwd(const float* cur, int upsample, float half_range, float step,
                           const float* step_dev, float* out, int B, int D, int h, int w,
                           void* stream);
int casmvs_warp_cost_ladder_fwd(const float* feats, const float* proj, const float* first_map,
                                const float* first_b, float first, const float* step_b, float step,
                                float* cost, int round_tf32, int B, int V, int C, int D, int h, int w,
                                int num_groups, void* stream);
int casmvs_regress_ladder_fwd(const float* logits, const float* first_map, const float* first_b,
                              float first, const float* step_b, float step, float* depth,
                              float* confidence, int64_t* index, int B, int D, int h, int w,
                              void* stream);

/* ---- FeatureNet top-down path, fused (adjacent to the hot path; SURVEY.md §8f-2) ----
 * One pyramid level of models/mvsnet.py:36-52:
 *   feat = upsample_x2_bilinear(prev, align_corners=True) + conv1x1(c, lat_w) + lat_b   (32 ch)
 *   out  = conv3x3(feat, smooth_w, pad 1) + smooth_b
 * prev (N,h/2,w/2,32), c (N,h,w,CLAT), out (N,h,w,COUT), feat_out (N,h,w,32) or NULL; all
 * channels-last.  lat_w (32,CLAT[,1,1]) and smooth_w (COUT,32,3,3) in torch layout. */
int casmvs_fpn_level_fwd(const float* prev, const float* c, const float* lat_w,
                         const float* lat_b, const float* smooth_w, const float* smooth_b,
                         float* feat_out, float* out, int N, int h, int w, int CLAT, int COUT,
                         void* stream);

/* The same level split in two for the tensor-core path: this call produces
 *   feat = upsample_x2_bilinear(prev, align_corners=True) + conv1x1(c, lat_w) + lat_b
 * (N,h,w,32), optionally TF32-rounded, and the 3x3 smooth runs as a CASMVS_CONV_PLANAR
 * casmvs_conv3d_fwd on wgmma.  prev == NULL: feat = conv1x1(c) + lat_b (the `toplayer`,
 * mvsnet.py:27,41).  lat_w (32,CLAT[,1,1]) torch layout; CLAT % 4 == 0. */
int casmvs_fpn_merge_fwd(const float* prev, const float* c, const float* lat_w,
                         const float* lat_b, float* feat, int N, int h, int w, int CLAT,
                         int round_tf32, void* stream);

/* First FeatureNet block (ConvBnReLU(3, 8, 3, 1, 1), mvsnet.py:13 + modules.py:8-18) with the
 * eval-mode ABN folded: y = LeakyReLU(conv3x3(x, w, pad 1) + bias).  x (N,3,H,W) planar fp32
 * (the image batch as the data loader hands it over, no re-layout), w (8,3,3,3) torch
 * layout already multiplied by the ABN scale, y (N,H,W,8) channels-last. */
int casmvs_conv2d_rgb8_fwd(const float* x, const float* w, const float* bias, float slope,
                           float* y, int N, int H, int W, int round_tf32, void* stream);

/* The 5x5 stride-2 blocks of FeatureNet (ConvBnReLU(8,16,5,2,2) / (16,32,5,2,2), mvsnet.py:16,20
 * + modules.py:8-18) with the eval-mode ABN folded, on wgmma (TF32 operands):
 *   y = LeakyReLU(conv5x5_s2_p2(x, w) + shift)
 * x (N,H,W,Cin) channels-last, w (Cout,Cin,5,5) torch layout already multiplied by the ABN
 * scale, y (N,(H-1)/2+1,(W-1)/2+1,Cout) channels-last, optionally stored TF32-rounded.  The
 * operand image built from `w` is cached by pointer (casmvs_invalidate_weight_cache). */
int casmvs_conv2d_5x5s2_fwd(const float* x, const float* w, const float* shift, float slope,
                            float* y, int N, int Cin, int Cout, int H, int W, int round_tf32,
                            void* stream);

/* The same blocks in the fp32 precision mode: CUDA-core FMA, bit-faithful products, output
 * unrounded.  Same layouts; w is the plain (Cout,Cin,5,5) torch tensor (nothing is cached). */
int casmvs_conv2d_5x5s2_fp32_fwd(const float* x, const float* w, const float* shift, float slope,
                                 float* y, int N, int Cin, int Cout, int H, int W, void* stream);

/* In-place x[...,c] = LeakyReLU(x[...,c] + bias[c]) on a channels-last tensor (C % 4 == 0):
 * the epilogue of a folded conv + eval-mode ABN block (models/modules.py:8-18). */
int casmvs_bias_lrelu_nhwc(float* x, const float* bias, float slope, size_t numel, int C,
                           void* stream);
/* Same, optionally storing the result TF32-rounded (round to nearest) for a tensor-core
 * consumer that would otherwise truncate it. */
int casmvs_bias_act_nhwc(float* x, const float* bias, float slope, size_t numel, int C,
                         int round_tf32, void* stream);

/* ---- backward of the hot path (SURVEY.md 8 f-1; reference train.py:99-127) -----------------
 * casmvs_warp_cost_bwd: gradient of casmvs_warp_cost_fwd w.r.t. the features (the only
 * differentiable input: hypotheses are detached, models/mvsnet.py:231).  All tensors
 * channels-last: feats (B,V,h,w,C), grad_cost (B,D,h,w,Cout), grad_feats (B,V,h,w,C) which the
 * caller ZEROES first (the bilinear taps are scattered into it with atomics).
 * casmvs_conv3d_wgrad: grad_w[27][Ca][Cb] += sum_{b,o} x[b, stride*o + k - 1, a] * grad_y[b,o,b']
 * for Conv3d (x = layer input, grad_y = output gradient, Ca = Cin, Cb = Cout) and, with the
 * roles swapped (x = output gradient, grad_y = layer input, stride 2), for ConvTranspose3d;
 * caller zeroes grad_w.  Channels <= 64.  The DATA gradients are forward kernels:
 * conv s1 -> conv s1 with flipped/transposed weights, conv s2 -> CASMVS_CONV_TRANSPOSE,
 * transposed -> conv s2 (casmvs_conv3d_fwd, scale = shift = NULL, slope = 1).
 * casmvs_regress_bwd: grad_logits = softmax(logits) * (depth_values - depth) * grad_depth. */
int casmvs_warp_cost_bwd(const float* feats, const float* proj, const float* depth_values,
                         const float* grad_cost, float* grad_feats, int B, int V, int C, int D,
                         int h, int w, int num_groups, void* stream);
int casmvs_conv3d_wgrad(const float* x, const float* grad_y, float* grad_w, int B, int Ca, int Cb,
                        int Di, int hi, int wi, int Do, int ho, int wo, int stride, void* stream);
int casmvs_regress_bwd(const float* logits, const float* depth_values, int dv_is_vector,
                       const float* grad_depth, float* grad_logits, int B, int D, int h, int w,
                       void* stream);

/* ---- training loss and depth metrics (reference losses.py, metrics.py) ----------------------
 * Per level l < levels (<= 4): pred[l], gt[l] (B,h_l,w_l) float32, mask[l] (B,h_l,w_l) uint8
 * (bool; nonzero = valid); hw is a HOST array (levels,2) of (h_l, w_l); pred / gt / mask /
 * grad_pred are HOST arrays of device pointers.
 * casmvs_sl1_loss_fwd: loss (device float[1]) = sum_l 2^(1-l) * mean over the mask of
 *   smoothL1(pred_l - gt_l) (beta 1); an empty mask gives NaN.  metrics (device float[5]) =
 *   level 0's sum |e|, #(|e| < 1), #(|e| < 2), #(|e| < 4), n_0; counts (device int64[levels]) =
 *   n_l.  Any output may be NULL.  Sums are fp64 in a fixed order (bit-identical run to run),
 *   stored as fp32.  workspace: casmvs_sl1_loss_workspace_bytes() bytes of device memory.
 * casmvs_sl1_loss_bwd: grad_pred[l] (device, all pixels written) = the gradient of that loss
 *   given d(loss) = *grad_loss (device float) and the forward's counts, in ATen's operation
 *   order (bit-identical to autograd of the reference's loss); 0 outside the mask. */
size_t casmvs_sl1_loss_workspace_bytes(void);
int casmvs_sl1_loss_fwd(const float* const* pred, const float* const* gt,
                        const uint8_t* const* mask, const int* hw, int B, int levels, float* loss,
                        float* metrics, long long* counts, void* workspace, size_t workspace_bytes,
                        void* stream);
int casmvs_sl1_loss_bwd(const float* const* pred, const float* const* gt,
                        const uint8_t* const* mask, const int* hw, int B, int levels,
                        const long long* counts, const float* grad_loss, float* const* grad_pred,
                        void* stream);

/* ---- input pipeline (SURVEY.md 8 f-4) -------------------------------------
 * T.ToTensor() + T.Normalize(mean, std) of the reference's data sets (datasets/dtu.py:130-137)
 * for images uploaded as bytes: images (N,H,W,3) uint8 RGB -> out (N,3,H,W) float32,
 * y = ((float)x / 255 - mean[c]) / std[c] in that operation order (bit-identical to
 * torchvision).  mean3 / std3 are HOST arrays of 3 floats.  H*W % 4 == 0 when N > 1. */
int casmvs_normalize_u8_fwd(const uint8_t* images, float* out, int N, int H, int W,
                            const float* mean3, const float* std3, void* stream);

/* Resamplers of the scan readers, byte-identical to the host libraries the reference uses:
 * images (N,H,W,3) uint8 -> out (N,OH,OW,3) uint8.  The weight tables are DEVICE int32 arrays
 * the caller computes once per (H,W) -> (OH,OW) pair (casmvsnet_pl_b200/io.py).
 * casmvs_resize_u8_pil_fwd: Pillow Image.resize(size, BILINEAR) (datasets/tanks.py:134-135,
 *   blendedmvs.py:161-163, dtu.py:159-162).  Horizontal pass (skipped when OW == W) then vertical
 *   pass (skipped when OH == H), each out = clip8(((1 << 21) + sum_k in[lo + k] * coef[k]) >> 22);
 *   xbounds (OW,2) / ybounds (OH,2) = (lo, taps), xcoef (OW,xks) / ycoef (OH,yks) = Pillow's
 *   22-bit coefficients.  Tables of a skipped pass may be NULL; tmp (N,H,OW,3) holds the
 *   intermediate and is needed only when both passes run.  Same size: a device copy.
 * casmvs_resize_u8_linear_fwd: cv2.resize(..., INTER_LINEAR) of 8-bit images (eval.py:266-268),
 *   per channel, so BGR and RGB input give the same bytes.  xtab (OW,4) / ytab (OH,4) =
 *   (i0, i1, w0, w1) with 11-bit weights, 16-byte aligned; h = in[i0]*w0 + in[i1]*w1 along x,
 *   out = (((w0*(h0>>4))>>16) + ((w1*(h1>>4))>>16) + 2) >> 2 along y. */
int casmvs_resize_u8_pil_fwd(const uint8_t* images, uint8_t* out, uint8_t* tmp, int N, int H,
                             int W, int OH, int OW, const int* xbounds, const int* xcoef, int xks,
                             const int* ybounds, const int* ycoef, int yks, void* stream);
int casmvs_resize_u8_linear_fwd(const uint8_t* images, uint8_t* out, int N, int H, int W, int OH,
                                int OW, const int* xtab, const int* ytab, void* stream);

/* ---- geometric-consistency filter + refinement + back-projection (SURVEY.md 8 f-3) ------
 * One reference view of eval.py:262-318 on the device; replaces xy_ref2src / xy_src2ref /
 * check_geo_consistency (eval.py:113-182, numba + cv2.remap on the CPU).  For every reference
 * pixel and each of the S source views: project with depth_ref, sample the source depth (and
 * image) bilinearly with cv2.remap's semantics (map rounded to 1/32 px, zero outside), lift
 * back, mask = |dp| < 1 px and |dd|/d < 1 %.
 *   depth_ref (H,W); image_ref (H,W,3) or NULL; proba_ref (H/4,W/4) or NULL (= confidence_2,
 *   upsampled x4 like cv2.resize INTER_LINEAR and compared with conf_thresh);
 *   depth_src / image_src: HOST arrays of S device pointers; proj_ref2src / proj_src2ref: HOST
 *   arrays (S,3,4) = (P_src @ inv(P_ref))[:3] / (P_ref @ inv(P_src))[:3]; ref2world (4,4) device.
 * Outputs (device): depth_refined (H,W) = (depth_ref + sum of consistent reprojections)/(n+1),
 * image_refined (H,W,3) or NULL, geo_count (H,W) int32, mask_final (H,W) uint8 or NULL
 * (geo_count >= min_consistent and confidence), points (H,W,3) world coordinates of the
 * refined depth or NULL; reproj_dbg (S,H,W) / mask_dbg (S,H,W) per-view results or NULL. */
int casmvs_geo_fuse_fwd(const float* depth_ref, const float* image_ref, const float* proba_ref,
                        const float* const* depth_src, const float* const* image_src,
                        const float* proj_ref2src, const float* proj_src2ref,
                        const float* ref2world, int S, int H, int W, float conf_thresh,
                        int min_consistent, float* depth_refined, float* image_refined,
                        int* geo_count, unsigned char* mask_final, float* points,
                        float* reproj_dbg, unsigned char* mask_dbg, void* stream);

/* ---- DTU point-cloud scoring (reference evaluations/dtu, MATLAB)--------------------------
 * The two heavy steps of the DTU scorer on the device; the masks, statistics and the sort /
 * run-length scan that turn cell keys into cells are torch ops (casmvsnet_pl_b200/dtu_eval.py).
 * points / targets / queries are (N,3) float32; cell lists are the sorted unique keys, with
 * cell_start (ncells+1) int32 offsets into the key-sorted points.
 *
 * casmvs_pcd_cell_keys: int64 cell key of each point for cells of edge `cell` with corner (0,0,0)
 *   at (ox,oy,oz), grid dims g < 2^20.  sub == 1: key = (ix*gy + iy)*gz + iz.  sub == 8: super
 *   cells of 8^3 cells first, key = ((sx*SY + sy)*SZ + sz) << 9 | lx << 6 | ly << 3 | lz with
 *   s = i >> 3, l = i & 7, S = ceil(g/8).  Points outside the grid (or NaN) get INT64_MAX.
 * Thinning (reducePts_haa.m): the kept set is the lexicographically-first maximal set of points
 *   pairwise more than `dst` apart for the visiting order `rank` (a permutation of 0..n-1), i.e.
 *   what visiting the points in rank order and keeping each point no kept point lies within dst
 *   of gives.  |p - q| <= dst is evaluated in double as (dx*dx + dy*dy) + dz*dz <= dst*dst.
 *   Points, rank and state are in key order of a sub == 1 grid whose cell edge is > dst.
 *   casmvs_pcd_thin_prepare fills the workspace (a 27-neighbour table per cell and the cell of
 *   each point); then call casmvs_pcd_thin_round, starting from state = 0 (undecided), until the
 *   device int *undecided it writes is 0.  state ends 1 (kept) or 2 (removed).
 * casmvs_pcd_capped_nn (MaxDistCP.m): dist[i] = min(nearest-target distance, cap) in double for a
 *   query with box_lo <= q < box_hi on every axis, cap otherwise.  Targets are in key order of a
 *   sub == 8 grid of edge h at origin3 that covers [box_lo - cap, box_hi + cap]; super_begin
 *   (prod(super_dims3)+1) int32 = index of the first cell of each super cell in the cell list.
 *   origin3, super_dims3, box_lo3, box_hi3 are HOST arrays of 3. */
int casmvs_pcd_cell_keys(const float* points, int n, double ox, double oy, double oz, double cell,
                         int gx, int gy, int gz, int sub, int64_t* keys, void* stream);
size_t casmvs_pcd_thin_workspace_bytes(int n, int ncells);
int casmvs_pcd_thin_prepare(const int64_t* cell_keys, const int* cell_start, int n, int ncells,
                            int gx, int gy, int gz, void* workspace, size_t workspace_bytes,
                            void* stream);
int casmvs_pcd_thin_round(const float* points, const int* rank, const int* cell_start, int n,
                          int ncells, double dst, unsigned char* state, int* undecided,
                          const void* workspace, size_t workspace_bytes, void* stream);
int casmvs_pcd_capped_nn(const float* queries, int nq, const float* targets,
                         const int64_t* cell_keys, const int* cell_start, int ncells,
                         const int* super_begin, const double* origin3, double h,
                         const int* super_dims3, const double* box_lo3, const double* box_hi3,
                         double cap, double* dist, void* stream);

/* ---- layout helpers ------------------------------------------------------ */
/* (N,C,S) -> (N,S,C) and back, S = product of spatial dims. */
int casmvs_nchw_to_nhwc(const float* in, float* out, int N, int C, size_t S, void* stream);
int casmvs_nhwc_to_nchw(const float* in, float* out, int N, int C, size_t S, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CASMVS_H_ */
