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

/* OR-ed into casmvs_costreg_fwd's precision: the caller does not read the workspace after the
 * call.  Where casmvs_costreg_tail_supported, conv11 and the prob head then run as one kernel
 * that computes the logits from u9 and c0 (the same logits, bit for bit), and u11 is never
 * stored.  Without it every activation c0 .. u11 is left in the workspace. */
#define CASMVS_FUSED_TAIL 1024

/* Inverse-depth plane sweep (README "Wide depth ranges"; the rule is stated in regress.cu).
 * OR-ed into casmvs_regress_fwd's input_is_prob: regress in 1/depth (depth = 1/sum p_d/dv_d).
 * OR-ed into casmvs_regress_bwd's dv_is_vector: the gradient of that regression.
 * OR-ed into casmvs_warp_cost_ladder_fwd's round_tf32: the ladder is in inverse depth, the
 * hypotheses are 1/(first - step*d) (first and step in 1/depth units). */
#define CASMVS_INVERSE_DEPTH 2048

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
/* 1 when a CASMVS_TF32 casmvs_conv3d_fwd of this layer runs on a tensor-core kernel, 0 when it
 * falls back to the CUDA cores.  A tensor-core kernel reads only the top 19 bits of each fp32
 * activation (it truncates), so a caller whose activations are not TF32-rounded rounds them
 * first where this is 1.  Host-only: no device is touched. */
int casmvs_conv3d_tensor_core(int Cin, int Cout, int kind, int stride, int has_skip);

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
 * 16-byte aligned: NHWC feats, the workspace (NCHW feats), an NHWC cost.
 */
size_t casmvs_warp_cost_workspace_bytes(int feat_layout, int B, int V, int C, int h, int w);
int casmvs_warp_cost_fwd(const float* feats, int feat_layout, const float* proj,
                         const float* depth_values, float* cost, int cost_layout,
                         int B, int V, int C, int D, int h, int w, int num_groups,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Stand-alone homo_warp (models/modules.py:52-92): materialises the warped
 * volume for API completeness.  src_feat (B,C,h,w)|(B,h,w,C), proj (B,3,4),
 * depth_values (B,D,h,w) -> warped (B,C,D,h,w)|(B,D,h,w,C).  src_feat and an
 * NHWC warped 16-byte aligned.                                             */
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
 * x 16-byte aligned; y and skip too when Cout > 1.
 * In the TF32 mode a layer shape that no tensor-core kernel covers runs on the CUDA cores
 * (casmvs_fallback_count).
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
 * accepts a CASMVS_BLOCKED input: TF32, and a tensor-core kernel covers every one of the 11
 * layers (conv1 .. prob always are; conv0 for Cin in {8,16,32}), else 0.  The other cases run
 * channels-last, layers no tensor-core kernel covers on the CUDA cores.
 * casmvs_costreg_fwd needs x and workspace 16-byte aligned. */
int casmvs_costreg_blocked_supported(int Cin, int precision);
int casmvs_costreg_fwd(const float* x, const float* params, float* logits,
                       int B, int Cin, int D, int h, int w, int precision,
                       void* workspace, size_t workspace_bytes, void* stream);
/* 1 when casmvs_costreg_fwd with CASMVS_FUSED_TAIL runs conv11 + prob as one kernel: where
 * casmvs_costreg_blocked_supported (the kernel reads and writes blocked activations). */
int casmvs_costreg_tail_supported(int Cin, int precision);
/* One step of casmvs_costreg_fwd, with its arguments (CASMVS_FUSED_TAIL ignored), for timing the
 * layers one at a time: layer 0 .. 10 runs that layer on the activations a full call leaves in
 * the workspace; layer 11 runs the fused conv11 + prob kernel (u9, c0 -> logits), where
 * casmvs_costreg_tail_supported. */
int casmvs_costreg_layer_fwd(const float* x, const float* params, float* logits,
                             int B, int Cin, int D, int h, int w, int precision,
                             void* workspace, size_t workspace_bytes, int layer, void* stream);

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
 * casmvs_warp_cost_ladder_fwd: channels-last features and cost volume, both 16-byte aligned;
 * shapes of the staged kernel only (casmvs_warp_cost_ladder_supported), error otherwise.
 * round_tf32: nonzero = store the cost TF32-rounded; | CASMVS_BLOCKED = store it blocked,
 * (B,Cout/4,D,h,w,4), for casmvs_costreg_fwd with CASMVS_BLOCKED.
 * casmvs_warp_cost_ladder_supported: 1 when the staged kernel covers the shape (V-1 in {1,2},
 * C in {8,16,32}, num_groups 1 or 8) and CASMVS_K1_SMEM=0 does not send every shape to the
 * gather kernel, else 0. */
int casmvs_depth_first_fwd(const float* cur, int upsample, float half_range, float step,
                           const float* step_dev, float* out, int B, int D, int h, int w,
                           void* stream);
int casmvs_warp_cost_ladder_supported(int V, int C, int num_groups);
int casmvs_warp_cost_ladder_fwd(const float* feats, const float* proj, const float* first_map,
                                const float* first_b, float first, const float* step_b, float step,
                                float* cost, int round_tf32, int B, int V, int C, int D, int h, int w,
                                int num_groups, void* stream);
int casmvs_regress_ladder_fwd(const float* logits, const float* first_map, const float* first_b,
                              float first, const float* step_b, float step, float* depth,
                              float* confidence, int64_t* index, int B, int D, int h, int w,
                              void* stream);

/* ---- inverse-depth forms (CASMVS_INVERSE_DEPTH) -----------------------------------------
 * casmvs_inverse_hypotheses_fwd: planes evenly spaced in 1/depth, d_k = 1/(u_0 - step*k).
 * cur == NULL: the coarsest stage, u_0 = u_first; planes must be D.
 * cur (B,h/2,w/2): a finer stage; cur is upsampled x2 as in casmvs_depth_hypotheses_fwd and
 * u_0 = max(1/c + (D/2)*step, u_far + (D-1)*step).  planes == D writes the depths (B,D,h,w);
 * planes == 1 writes u_0 (B,h,w), the first rung of an inverse ladder.
 * u_first_dev, u_far_dev, step_dev: (B) device values that override the scalars when non-NULL.
 * casmvs_regress_ladder_inverse_fwd: casmvs_regress_ladder_fwd over the inverse ladder
 * 1/(first - step*d), with the inverse regression. */
int casmvs_inverse_hypotheses_fwd(const float* cur, float u_first, const float* u_first_dev,
                                  float u_far, const float* u_far_dev, float step,
                                  const float* step_dev, float* out, int planes, int B, int D,
                                  int h, int w, void* stream);
int casmvs_regress_ladder_inverse_fwd(const float* logits, const float* first_map,
                                      const float* first_b, float first, const float* step_b,
                                      float step, float* depth, float* confidence, int64_t* index,
                                      int B, int D, int h, int w, void* stream);

/* ---- adaptive depth ranges (README "Adaptive depth ranges"; the rule is stated in regress.cu)
 * casmvs_adaptive_hypotheses_fwd: the planes of a finer stage from the previous stage's depth
 * cur and spread, both (B,h/2,w/2), upsampled x2 as in casmvs_depth_hypotheses_fwd:
 * r = max(1.5*s, step), lo = max(c - r, 1e-7), hi = c + r, pstep = (hi - lo)/(D-1), plane k =
 * lo + pstep*k.  step: the uniform plane step g of the stage, step_dev (B) overrides it when
 * non-NULL.  planes == D writes the planes (B,D,h,w) to out; planes == 1 writes lo to out and
 * pstep to step_out, both (B,h,w).  D >= 2.
 * casmvs_regress_spread_fwd: casmvs_regress_fwd (uniform regression; input_is_prob 0 or 1) that
 * also writes spread (B,h,w) = sqrt(sum_d p_d (dv_d - depth)^2).  depth, confidence, index and
 * prob are the bits casmvs_regress_fwd writes.
 * casmvs_regress_ladder_spread_fwd: casmvs_regress_ladder_fwd with the spread.  step_map (B,h,w)
 * non-NULL: the per-pixel-step ladder first_map + step_map*d (first_b, first, step_b and step
 * are ignored), and spread may be NULL.
 * casmvs_warp_cost_ladder_step_fwd: casmvs_warp_cost_ladder_fwd over the per-pixel-step ladder
 * first_map + step_map*d; round_tf32 takes 1 and CASMVS_BLOCKED. */
int casmvs_adaptive_hypotheses_fwd(const float* cur, const float* spread, float step,
                                   const float* step_dev, float* out, float* step_out, int planes,
                                   int B, int D, int h, int w, void* stream);
int casmvs_regress_spread_fwd(const float* logits, const float* depth_values, int dv_is_vector,
                              int input_is_prob, float* depth, float* confidence, int64_t* index,
                              float* prob, float* spread, int B, int D, int h, int w,
                              void* stream);
int casmvs_regress_ladder_spread_fwd(const float* logits, const float* first_map,
                                     const float* first_b, float first, const float* step_b,
                                     float step, const float* step_map, float* depth,
                                     float* confidence, int64_t* index, float* spread, int B,
                                     int D, int h, int w, void* stream);
int casmvs_warp_cost_ladder_step_fwd(const float* feats, const float* proj, const float* first_map,
                                     const float* step_map, float* cost, int round_tf32, int B,
                                     int V, int C, int D, int h, int w, int num_groups,
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

/* ---- deterministic backward: the same bits for the same inputs, shapes and device model ------
 * casmvs_warp_cost_bwd_det: what casmvs_warp_cost_bwd computes, with no float atomics.  A
 *   contribution pass records every bilinear tap's destination texel, weight and coefficient; a
 *   stable radix sort groups them by destination; each texel then adds its contributions in
 *   contribution order.  The reference view's gradient is summed over all D planes by one
 *   thread.  grad_feats is WRITTEN (no zeroing needed).  Same arguments and dims as
 *   casmvs_warp_cost_bwd, plus `workspace` (256-byte aligned) of at least
 *   casmvs_warp_cost_bwd_det_workspace_bytes(B, V, C, D, h, w) bytes: 4 (C + 20) bytes per
 *   (batch item, plane, pixel, source view) plus the sort's temporary storage (0 = dims out of
 *   range).  feats and grad_feats need 16-byte alignment.
 * casmvs_conv3d_wgrad_det: what casmvs_conv3d_wgrad computes; each voxel chunk stores its
 *   [27][Ca][Cb] partial to the workspace and a second kernel adds the chunks in chunk order.
 *   The chunking depends on B * Do * ho * wo only.  grad_w is WRITTEN.  workspace: at least
 *   casmvs_conv3d_wgrad_det_workspace_bytes(B, Ca, Cb, Do, ho, wo) bytes.
 * casmvs_upsample2x_bilinear_bwd: grad_x (N,C,h,w) of y = bilinear upsample to (2h, 2w) with
 *   align_corners=True, given grad_y (N,C,2h,2w); both CASMVS_NCHW or both CASMVS_NHWC
 *   (`layout`).  Each input element gathers its output pixels in a fixed order with ATen's
 *   weights.  grad_x is WRITTEN. */
size_t casmvs_warp_cost_bwd_det_workspace_bytes(int B, int V, int C, int D, int h, int w);
int casmvs_warp_cost_bwd_det(const float* feats, const float* proj, const float* depth_values,
                             const float* grad_cost, float* grad_feats, int B, int V, int C,
                             int D, int h, int w, int num_groups, void* workspace,
                             size_t workspace_bytes, void* stream);
size_t casmvs_conv3d_wgrad_det_workspace_bytes(int B, int Ca, int Cb, int Do, int ho, int wo);
int casmvs_conv3d_wgrad_det(const float* x, const float* grad_y, float* grad_w, int B, int Ca,
                            int Cb, int Di, int hi, int wi, int Do, int ho, int wo, int stride,
                            void* workspace, size_t workspace_bytes, void* stream);
int casmvs_upsample2x_bilinear_bwd(const float* grad_y, float* grad_x, int N, int C, int h, int w,
                                   int layout, void* stream);

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

/* ---- self-supervised photometric loss (csrc/photo_loss.cu has the full rule) ---------------
 * imgs (B,V,3,H,W) float32 normalised network input (view 0 = reference), proj_mats
 * (B,V-1,levels,3,4), depth_interval (B) float32, all device; depth / selection / grad_depth /
 * dbg_* are HOST arrays of `levels` device pointers to (B,H/2^l,W/2^l) maps (dbg_e: (B,V-1,h,w));
 * interval_ratios is a HOST float[levels].
 *   L = sum_l 2^(1-l) (P_l + smooth_weight S_l), P_l = mean over pixels with a valid source of
 *   the mean of the topk smallest 0.85 (1 - SSIM3x3) / 2 + 0.15 |L1| errors over the warped
 *   sources, S_l the edge-aware smoothness of depth / (depth_interval * interval_ratios[l]).
 * casmvs_photo_loss_fwd: loss (device float[1]), stats (device float[levels][3] = P_l, S_l,
 *   N_l), counts (device int64[levels] = N_l) and selection (uint16 per pixel, bit s = source
 *   s selected) for the backward.  dbg_e (NaN where (q, s) is not valid), dbg_valid (uint16
 *   bits) and dbg_lossq (NaN where no source is valid) may be NULL.  fp64 sums in a fixed order,
 *   no atomics: bit-identical run to run.  workspace: casmvs_photo_loss_workspace_bytes bytes.
 * casmvs_photo_loss_bwd: grad_depth[l] (every pixel written) = dL/d depth_l * (*grad_loss,
 *   device float), a gather that needs no host synchronisation.
 * Refused (status -1): V - 1 outside 1..16, topk outside 1..V-1, levels outside 1..4, a level
 * smaller than 3x3 or H, W not divisible by 2^(levels-1), smooth_weight not finite or < 0. */
size_t casmvs_photo_loss_workspace_bytes(int B, int H, int W, int levels);
int casmvs_photo_loss_fwd(const float* imgs, const float* proj_mats, const float* depth_interval,
                          const float* const* depth, const float* interval_ratios, int B, int V,
                          int H, int W, int levels, int topk, float smooth_weight,
                          uint16_t* const* selection, float* loss, float* stats, long long* counts,
                          float* const* dbg_e, uint16_t* const* dbg_valid, float* const* dbg_lossq,
                          void* workspace, size_t workspace_bytes, void* stream);
int casmvs_photo_loss_bwd(const float* imgs, const float* proj_mats, const float* depth_interval,
                          const float* const* depth, const float* interval_ratios, int B, int V,
                          int H, int W, int levels, int topk, float smooth_weight,
                          const uint16_t* const* selection, const long long* counts,
                          const float* grad_loss, float* const* grad_depth, void* stream);

/* ---- input pipeline (SURVEY.md 8 f-4) -------------------------------------
 * T.ToTensor() + T.Normalize(mean, std) of the reference's data sets (datasets/dtu.py:130-137)
 * for images uploaded as bytes: images (N,H,W,3) uint8 RGB -> out (N,3,H,W) float32,
 * y = ((float)x / 255 - mean[c]) / std[c] in that operation order (bit-identical to
 * torchvision).  mean3 / std3 are HOST arrays of 3 floats.  H*W % 4 == 0 when N > 1. */
int casmvs_normalize_u8_fwd(const uint8_t* images, float* out, int N, int H, int W,
                            const float* mean3, const float* std3, void* stream);
/* The same conversion after T.ColorJitter(brightness, contrast) on the PIL image (the training
 * transform of datasets/blendedmvs.py:130-137), bit-identical to torchvision + Pillow.
 * jitter: DEVICE (N,3) float32 per image = (brightness_first != 0, b, c): brightness is
 * Image.blend(black, img, b), contrast Image.blend(gray(m), img, c) with m = int(mean L + 0.5)
 * of the image as it stands when contrast is applied.  lsum: DEVICE scratch of N int64 (8-byte
 * aligned), zeroed here.  No host synchronisation: graph-capturable.  H*W % 4 == 0 when N > 1. */
int casmvs_jitter_normalize_u8_fwd(const uint8_t* images, const float* jitter, float* out,
                                   long long* lsum, int N, int H, int W, const float* mean3,
                                   const float* std3, void* stream);

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

/* Undistortion of distorted COLMAP views (casmvsnet_pl_b200/colmap.py undistorted_camera):
 * images (N,H,W,3) uint8 of one source camera -> out (N,OH,OW,3) uint8 in its undistorted
 * PINHOLE camera.  model: COLMAP's model id (0-6, 8, 9; FOV and THIN_PRISM_FISHEYE are refused);
 * src_params: HOST array of the model's parameters in COLMAP's order; dst_params: HOST array
 * (fx, fy, cx, cy) of the undistorted camera.  Both are copied into the launch, not to the device.
 * Per output pixel, in float64 with every operation rounded separately: u = (x + 0.5 - cx') / fx',
 * v likewise, COLMAP's forward distortion and projection to (X, Y), sx = X - 0.5, sy = Y - 0.5;
 * 0 when either lies more than 1e-6 outside [0, W-1] / [0, H-1], else the bilinear sample at
 * the clamped point, rounded by floor(s + 0.5).  The map is computed once per output pixel and
 * applied to all N images.  H, W >= 2. */
int casmvs_undistort_u8_fwd(const uint8_t* images, uint8_t* out, int N, int H, int W, int OH,
                            int OW, int model, const double* src_params, const double* dst_params,
                            void* stream);

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

/* ---- dynamic consistency fusion ---------------------------------------------------------
 * casmvs_geo_fuse_fwd with the count-based dynamic consistency check of D2HC-RMVSNet (Yan et
 * al., ECCV 2020) in place of the fixed one: the same arguments without min_consistent, the
 * same projection, sampling and back-projection, and per source the same fp32 errors
 * e_pix = dx*dx + dy*dy and e_dep = |(rz - d) / d|.  Source s is consistent at level k
 * (k = 2..10) when e_pix < (k/4)^2 and e_dep < T_k = float32(k / 1300), computed in double and
 * rounded once; k_s is its least such level, 0 when there is none (NaN compares false).  With
 * n_k = #{s : 0 < k_s <= k}, the geometric mask holds when n_k >= k for some 2 <= k <= min(10, S)
 * (never when S < 2); mask_final is that AND the confidence test.  depth_refined, image_refined
 * and geo_count average and count the sources with k_s > 0, in source order.  reproj_dbg holds rz
 * for those sources, else 0; level_dbg (S,H,W) uint8 or NULL holds k_s.  Same checks as above:
 * S <= 16, dims, null pointers, proba needs H, W % 4 == 0. */
int casmvs_geo_fuse_dynamic_fwd(const float* depth_ref, const float* image_ref,
                                const float* proba_ref, const float* const* depth_src,
                                const float* const* image_src, const float* proj_ref2src,
                                const float* proj_src2ref, const float* ref2world, int S, int H,
                                int W, float conf_thresh, float* depth_refined,
                                float* image_refined, int* geo_count, unsigned char* mask_final,
                                float* points, float* reproj_dbg, unsigned char* level_dbg,
                                void* stream);

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
/* casmvs_pcd_capped_nn_index: casmvs_pcd_capped_nn that also writes index[i], the original index
 *   (target_index[k] of the key-sorted target k) of the nearest target, or -1 with dist = cap
 *   when no target lies strictly closer than cap.  d^2 = (dx*dx + dy*dy) + dz*dz, dx = t - q, in
 *   double from the float32 coordinates with every operation rounded to nearest (no
 *   contraction); dist = sqrt(d^2).  An exact tie goes to the lower original index. */
int casmvs_pcd_capped_nn_index(const float* queries, int nq, const float* targets,
                               const int64_t* cell_keys, const int* cell_start, int ncells,
                               const int* super_begin, const double* origin3, double h,
                               const int* super_dims3, const double* box_lo3,
                               const double* box_hi3, double cap, const int64_t* target_index,
                               double* dist, int64_t* index, void* stream);

/* ---- Statistical outlier removal (casmvsnet_pl_b200/cloud_filter.py) -------------------------
 * Every double operation below is rounded to nearest, no contraction, in the order written.
 * casmvs_pcd_knn_mean: mean[point_index[i]] = m_i, the mean distance from point i to its k
 *   (1..64) nearest other points of the same cloud, for n > k points.  points are in key order of
 *   a sub == 8 grid of edge h at origin3 that holds every point (cell lists and super_begin as for
 *   casmvs_pcd_capped_nn); point_index (n int64) maps them back to the input order.  d(i, j) =
 *   sqrt((dx*dx + dy*dy) + dz*dz), dx = double(x_j) - double(x_i); the point itself is not its
 *   own neighbour but exact duplicates are, at 0.  m_i = (the k smallest d(i, j) summed left to
 *   right in ascending order) / k.  Boxes are widened by `pad` (>= 0; it must cover the rounding
 *   of the cell keys and of the box bounds at the cloud's coordinates) before they are pruned.
 *   The result is exact for every h.  origin3 and super_dims3 are HOST arrays of 3.
 * casmvs_pcd_sor_keep: the statistics and keep mask of n >= 2 mean distances.  With chunks of
 *   1024 values in order, workspace (casmvs_pcd_sor_workspace_bytes(n)) gets the chunk sums of
 *   the m_i, then those of (m_i - mu)^2; stats (3 doubles, device) = mu = (chunk sums summed left
 *   to right) / n, sigma = sqrt((the same for the squares) / (n - 1)) and the threshold
 *   t = mu + std_ratio * sigma (std_ratio finite, > 0).  mask[i] = m_i <= t, and block_counts
 *   (casmvs_tnt_crop_blocks(n) ints) the kept count of each block, as casmvs_tnt_compact takes
 *   them.  No float atomics: two runs give the same bits. */
int casmvs_pcd_knn_mean(const float* points, int n, int k, const int64_t* cell_keys,
                        const int* cell_start, int ncells, const int* super_begin,
                        const double* origin3, double h, const int* super_dims3, double pad,
                        const int64_t* point_index, double* mean, void* stream);
size_t casmvs_pcd_sor_workspace_bytes(int n);
int casmvs_pcd_sor_keep(const double* mean, int n, double std_ratio, double* stats,
                        unsigned char* mask, int* block_counts, void* workspace,
                        size_t workspace_bytes, void* stream);

/* ---- Tanks and Temples scoring (casmvsnet_pl_b200/tnt_eval.py) ------------------------------
 * Every double operation below is rounded to nearest, no contraction, in the order written.
 * casmvs_tnt_transform_crop: out[i] = p_i, or with T (a HOST array of 12 doubles, rows 0..2 of a
 *   4x4, row-major) out[i].r = float32(((T_r0 x + T_r1 y) + T_r2 z) + T_r3) in double.  With axis
 *   0, 1 or 2 (the crop's orthogonal axis; -1 = no crop) it also writes mask[i] = 1 when out[i]
 *   lies in the crop volume (Open3D's CropInPolygon, in double): axis_min <= p[axis] <= axis_max
 *   and, with (u, v) = (y, z), (x, z) or (x, y), an odd number of polygon edges (i, j = i+1 mod m)
 *   with (P_i.u < p.u <= P_j.u) or (P_j.u < p.u <= P_i.u) whose node
 *   P_i.v + ((p.u - P_i.u) / (P_j.u - P_i.u)) * (P_j.v - P_i.v) is < p.v.  polygon is (m,2)
 *   doubles (u, v) on the DEVICE.  block_counts (casmvs_tnt_crop_blocks(n) ints) gets the kept
 *   points of each block of the launch.
 * casmvs_tnt_compact: the points with mask[i] != 0 in input order, given block_offsets, the int64
 *   exclusive scan of block_counts; out_index (optional) gets their input indices.
 * casmvs_tnt_voxel_mean: out[v] = float32(sum / count) of the points order[voxel_start[v]] ..
 *   order[voxel_start[v+1] - 1], summed per axis in double in that order.
 * casmvs_tnt_icp_moments: with s = src[i], t = tgt[index[i]] over the i with index[i] >= 0,
 *   s' = s - origin, t' = t - origin: moments (18 doubles, DEVICE) = count, sum |t - s|^2, sum s'
 *   (3), sum t' (3), sum |s'|^2, sum t'_a s'_b (3x3 row-major).  The sums are the same bits on
 *   every call: a grid fixed by n, a fixed reduction tree, no atomics.  origin3 is a HOST array. */
int casmvs_tnt_crop_blocks(int n);
int casmvs_tnt_transform_crop(const float* points, int n, const double* T, int axis,
                              double axis_min, double axis_max, const double* polygon,
                              int n_polygon, float* out, unsigned char* mask, int* block_counts,
                              void* stream);
int casmvs_tnt_compact(const float* points, const unsigned char* mask, int n,
                       const int64_t* block_offsets, float* out, int64_t* out_index, void* stream);
int casmvs_tnt_voxel_mean(const float* points, const int64_t* order, const int* voxel_start,
                          int n_voxels, float* out, void* stream);
size_t casmvs_tnt_icp_workspace_bytes(int n);
int casmvs_tnt_icp_moments(const float* src, int n, const float* tgt, const int64_t* index,
                           const double* origin3, double* moments, void* workspace,
                           size_t workspace_bytes, void* stream);

/* ---- view selection of a sparse reconstruction (casmvsnet_pl_b200/colmap.py) ---------------
 * casmvs_view_scores_fwd: the MVSNet paper's (section 4.1) view-selection scores, in double:
 *   scores[i][j] = sum over the points p that both images i and j see of G(theta_ij(p)),
 *   theta_ij(p) = degrees(acos(clamp(dot(unit(c_i - p), unit(c_j - p)), -1, 1))),
 *   G(theta) = exp(-(theta - 5)^2 / 2) for theta <= 5, exp(-(theta - 5)^2 / 200) else;
 *   a point on a camera centre contributes 0.  scores (n_img, n_img) is WRITTEN, symmetric, 0 on
 *   the diagonal.  centres (n_img,3) and points (n_pts,3) row-major doubles; the tracks in CSR
 *   form: point p is seen by track_img[track_ptr[p] .. track_ptr[p+1]) (int64 offsets, int32
 *   image ids).  The images of one track must be distinct; a pair with an id outside
 *   [0, n_img) contributes nothing.  n_img <= 65535.
 *   Deterministic: each score is added in ascending point order (pairs are expanded, stably
 *   radix-sorted by image pair and summed run by run), so the result is the same bits on every
 *   call and for every workspace size.  The pairs are processed in chunks of at most
 *   max_chunk_pairs entries (default 2^22); the chunk is the largest the workspace holds.
 *   The call synchronises `stream` once, to read the number of pairs (not graph-capturable).
 *   No points or fewer than two images: scores is zeroed, no kernel runs, workspace may be NULL.
 * casmvs_view_scores_workspace_bytes: the workspace (256-byte aligned) for chunks of at most
 *   max_chunk_pairs pairs (<= 0: the default, the fastest); 0 when none is needed. */
size_t casmvs_view_scores_workspace_bytes(int n_img, int n_pts, long long max_chunk_pairs);
int casmvs_view_scores_fwd(const double* centres, const double* points, const long long* track_ptr,
                           const int* track_img, int n_img, int n_pts, double* scores,
                           void* workspace, size_t workspace_bytes, void* stream);

/* ---- TSDF fusion and marching cubes (casmvsnet_pl_b200/mesh.py) -----------------------------
 * A sparse volume of bricks of 8^3 voxels; voxel ijk is centred at ijk * voxel (world units).
 * Brick (bx,by,bz) has key ((bx + 2^20) << 42) | ((by + 2^20) << 21) | (bz + 2^20), valid for
 * -2^20 <= b <= 2^20 - 2.  `keys` is the sorted, unique key list of the allocated bricks (nb
 * entries, nb <= 2^31 / 1536); voxel v = 512 * brick + (lz * 8 + ly) * 8 + lx, local lx = i - 8 bx.
 * Per voxel: tsdf (nb*512) f32, weight (nb*512) f32 (a view count), color (nb*512,3) f32.
 * casmvs_mesh_brick_keys: for each of n points (n,3) f32, the 8 keys (n,8) int64 of the bricks
 *   holding voxel centres in the cube of half-size trunc around it, per axis indices
 *   ceil((p - trunc)/voxel) .. floor((p + trunc)/voxel) (float, rounded division); a point
 *   spanning fewer than 2 bricks on an axis repeats the lower one.  NaN points and points whose
 *   bricks leave the packable range get INT64_MAX 8 times and add 1 to *dropped (device u64,
 *   not zeroed here).  voxel <= trunc <= 4 voxel.
 * casmvs_mesh_brick_neighbors: nbr (nb,7) int32, nbr[b][dx + 2dy + 4dz - 1] = index of brick
 *   b + (dx,dy,dz) for (dx,dy,dz) in {0,1}^3 \ 0, by binary search; -1 if not allocated.
 * casmvs_mesh_integrate: Curless & Levoy's projective TSDF of n_views masked depth maps (H,W) f32
 *   (0 = no depth) with colours image (H,W,3) f32, in view order; depth / image are HOST arrays
 *   of device pointers, proj a HOST array (n_views,4,4) f32 of world -> pixel matrices P.  Every
 *   voxel centre X and view, with every float operation rounded to nearest, no contraction:
 *     z  = ((P20 X + P21 Y) + P22 Z) + P23, likewise uz (row 0) and vz (row 1); skip unless z > 0
 *     px = floor(uz / z + 0.5), py = floor(vz / z + 0.5); skip outside the image or if D = 0
 *     sdf = D - z; skip unless sdf >= -trunc;  t = min(1, sdf / trunc)
 *     tsdf = (tsdf * w + t) / (w + 1);  color_c = (color_c * w + image_c) / (w + 1);  w = w + 1
 *   One thread per voxel, views batched 8 per launch: deterministic, no atomics.  The volume is
 *   not cleared: start from zeros.
 * Marching cubes over the cells (lower corner v, corners v + {0,1}^3) whose 8 corners are
 * allocated with weight > 0; a corner is inside when tsdf < 0; the case table is
 * csrc/mc_table.h (generated, see casmvsnet_pl_b200/mc_table.py).  Voxel v owns the edges
 * e = 3v + axis from v to v + unit(axis).
 * casmvs_mesh_count: cases (nb*512) u8 and tri_count (nb*512) int32 per cell (0 when not meshed);
 *   edge_used (nb*512*3) int32 = 1 for the crossing edges of meshed cells, else 0 (zeroed here).
 * casmvs_mesh_vertices: with edge_scan = inclusive scan of edge_used, the vertex of used edge q is
 *   number edge_scan[q] - 1: along the axis, t = s0 / (s0 - s1) of the end values in double,
 *   position (index + t) * voxel in double rounded once to f32 (other axes index * voxel);
 *   colour c0 + t (c1 - c0) in double, rint (half even), clamped to 0..255.  verts (N,3) f32,
 *   vcolor (N,3) u8.
 * casmvs_mesh_faces: with tri_scan = inclusive scan of tri_count, the triangles of cell v in table
 *   order from row tri_scan[v] - tri_count[v] of faces (M,3) int32 (vertex numbers); counter-
 *   clockwise seen from outside (the normal points from tsdf < 0 towards tsdf >= 0).
 * Empty volumes (nb = 0) launch nothing. */
int casmvs_mesh_brick_keys(const float* points, int n, float voxel, float trunc, long long* keys,
                           unsigned long long* dropped, void* stream);
int casmvs_mesh_brick_neighbors(const long long* keys, int nb, int* nbr, void* stream);
int casmvs_mesh_integrate(const long long* keys, int nb, float voxel, float trunc,
                          const float* const* depth, const float* const* image, const float* proj,
                          int n_views, int H, int W, float* tsdf, float* weight, float* color,
                          void* stream);
int casmvs_mesh_count(const int* nbr, int nb, const float* tsdf, const float* weight,
                      unsigned char* cases, int* tri_count, int* edge_used, void* stream);
int casmvs_mesh_vertices(const long long* keys, const int* nbr, int nb, float voxel,
                         const float* tsdf, const float* color, const int* edge_used,
                         const int* edge_scan, float* verts, unsigned char* vcolor, void* stream);
int casmvs_mesh_faces(const int* nbr, int nb, const unsigned char* cases, const int* tri_count,
                      const int* tri_scan, const int* edge_scan, int* faces, void* stream);

/* ---- Poisson surface reconstruction (csrc/poisson.cu, casmvsnet_pl_b200/poisson.py) ---------
 * A dense grid of N^3 nodes (N a power of two, 8..1024), spacing h; local node (x,y,z) is the
 * global node lo + (x,y,z) at world (lo + x) h; dense fields are flat, index (x N + y) N + z.  A
 * point p's cell is the node round(p / h) (float division, half to even); its splat corners are
 * floor(p / h) + {0,1}^3 with float32 weights (wx wy) wz, w = frac or 1 - frac, frac =
 * p / h - floor(p / h).  No float atomics: every sum has a fixed order.
 * casmvs_poisson_cell_keys: keys (n) int64 = flat local cell index, INT64_MAX for a point that is
 *   not finite, lies outside the grid, or (normals != NULL) has a zero-length or non-finite
 *   normal; unit_normals (n,3) f32 = normals / |normals| computed in double (0 when dropped).
 * casmvs_poisson_cell_moments: cells are runs of equal keys in the sorted points; cell_start
 *   (n_cells + 1) int32 offsets.  moments (n_cells,10) f64 = count, sum d, sum d d^T (xx, xy, xz,
 *   yy, yz, zz), d = p - (cx,cy,cz), summed in point order.
 * casmvs_poisson_cell_normals: cell_of (N^3) int32 = cell number of a node, -1 if empty; per cell,
 *   the moments of the 3x3x3 cells around it (x-major order) give the covariance; cell_normals
 *   (n_cells,3) f64 = unit eigenvector of its smallest eigenvalue (Jacobi, double); cell_ok = 0
 *   when the block holds < 3 points or lambda_mid <= 1e-10 lambda_max.
 * casmvs_poisson_orient: normals (n,3) f32 = the point's cell normal (point_cell (n) int32),
 *   flipped so that n . (C - p) > 0 for the nearest camera centre C of cams (n_cams,3) f64 on the
 *   device (ties to the lower index; a dot product of 0 keeps the sign).
 * casmvs_poisson_splat: one thread per node gathers the sorted points of the 27 cells around it:
 *   V (N^3,3) = sum w n, W (N^3) = sum w, C (N^3,3) = sum w rgb (rgb (n,3) u8, NULL = white),
 *   summed in double in cell and point order, stored f32.
 * casmvs_poisson_rhs: b (N^3) f32 = div V by central differences / (2h) at interior nodes, 0 on
 *   the outer layer; *bb (device f64) = sum of b^2.  workspace: casmvs_poisson_workspace_bytes(N^3).
 * Multigrid for (sum of the 6 neighbours - 6 x) / h^2 = rhs.  Level l (0 = finest) has n = N >> l
 * nodes per axis stored, node I at fine node 2^l I.  Level 0 has x = 0 on its outer layer (indices
 * 0 and N - 1, interior 1..N-2).  A coarse level (l > 0) has x = 0 at index 0 and at index n, fine
 * index N on every coarse level; node n is not stored and reads as 0, so the interior is 1..n-1.
 * casmvs_poisson_residual: r (N^3) f32 = b - L chi computed in double from chi (N^3) f64 on level
 *   0, 0 on the outer layer; *rr (device f64) = sum of r^2 (before rounding).
 * casmvs_poisson_smooth: `sweeps` red-black Gauss-Seidel sweeps (red: x+y+z even, first) on e
 *   (n^3) f32 of level `level` with right-hand side r at spacing h; zero_first: start from e = 0.
 * casmvs_poisson_mg_residual: out = r - L e (f32) at the level's interior nodes, 0 elsewhere.
 * casmvs_poisson_restrict: coarse (nf/2)^3 = full weighting of fine at coarse interior node I
 *   (1..nf/2-1; fine 2I + {-1,0,1}^3, weights (1/4,1/2,1/4)^3), 0 elsewhere.
 * casmvs_poisson_prolong_add: the interior nodes of fine (level fine_level, (2nc)^3) += trilinear
 *   interpolation of coarse (nc^3), coarse node I at fine 2I, coarse index nc counting as 0.
 * casmvs_poisson_accumulate: chi (f64) += e (f32).
 * casmvs_poisson_iso_sum: *sum (device f64) = sum over the points of chi trilinearly interpolated;
 *   a corner outside the grid counts as chi = 0 (poisson.py's grid keeps every corner inside).
 * casmvs_poisson_trim: keep (N^3) u8 = 1 where the 5x5x5 box around the node holds W > 0;
 *   workspace N^3 bytes.
 * casmvs_poisson_brick_flags: flags (nb_x,nb_y,nb_z) u8 = 1 for the global bricks b0 + (i,j,k)
 *   (mesh.cu's 8^3 bricks, key floor(global node / 8)) that hold a kept node.
 * casmvs_poisson_fill_bricks: in mesh.cu's brick layout (keys sorted), weight = 1 and colour =
 *   box5(C) / box5(W) (sums in double) at kept nodes, weight 0 and colour 0 elsewhere.
 * casmvs_poisson_fill_tsdf: tsdf = chi - iso (double, rounded once) where weight > 0, else 0.
 * casmvs_poisson_workspace_bytes: the reduction workspace for n terms. */
size_t casmvs_poisson_workspace_bytes(long long n);
int casmvs_poisson_cell_keys(const float* points, const float* normals, int n, float h, int lo_x,
                             int lo_y, int lo_z, int N, long long* keys, float* unit_normals,
                             void* stream);
int casmvs_poisson_cell_moments(const float* points, const int* cell_start, int n_cells, double cx,
                                double cy, double cz, double* moments, void* stream);
int casmvs_poisson_cell_normals(const long long* cell_keys, const int* cell_of,
                                const double* moments, int n_cells, int N, double* cell_normals,
                                unsigned char* cell_ok, void* stream);
int casmvs_poisson_orient(const float* points, const int* point_cell, const double* cell_normals,
                          int n, const double* cams, int n_cams, float* normals, void* stream);
int casmvs_poisson_splat(const float* points, const float* normals, const unsigned char* rgb,
                         const int* cell_start, const int* cell_of, int N, float h, int lo_x,
                         int lo_y, int lo_z, float* V, float* W, float* C, void* stream);
int casmvs_poisson_rhs(const float* V, int N, float h, float* b, double* workspace, double* bb,
                       void* stream);
int casmvs_poisson_residual(const double* chi, const float* b, int N, float h, float* r,
                            double* workspace, double* rr, void* stream);
int casmvs_poisson_smooth(float* e, const float* r, int n, int level, float h, int sweeps,
                          int zero_first, void* stream);
int casmvs_poisson_mg_residual(const float* e, const float* r, int n, int level, float h,
                               float* out, void* stream);
int casmvs_poisson_restrict(const float* fine, int nf, float* coarse, void* stream);
int casmvs_poisson_prolong_add(const float* coarse, int nc, float* fine, int fine_level,
                               void* stream);
int casmvs_poisson_accumulate(double* chi, const float* e, int N, void* stream);
int casmvs_poisson_iso_sum(const double* chi, const float* points, int n, int N, float h, int lo_x,
                           int lo_y, int lo_z, double* workspace, double* sum, void* stream);
int casmvs_poisson_trim(const float* W, int N, unsigned char* keep, unsigned char* workspace,
                        void* stream);
int casmvs_poisson_brick_flags(const unsigned char* keep, int N, int lo_x, int lo_y, int lo_z,
                               int b0_x, int b0_y, int b0_z, int nb_x, int nb_y, int nb_z,
                               unsigned char* flags, void* stream);
int casmvs_poisson_fill_bricks(const long long* keys, int nb, const unsigned char* keep,
                               const float* W, const float* C, int N, int lo_x, int lo_y, int lo_z,
                               float* weight, float* color, void* stream);
int casmvs_poisson_fill_tsdf(const long long* keys, int nb, const float* weight, const double* chi,
                             double iso, int N, int lo_x, int lo_y, int lo_z, float* tsdf,
                             void* stream);

/* ---- screened Poisson (the point-weight term; poisson.py's point_weight > 0) ----------------
 * A point's splat cell is its floor corner floor(p / h) - lo; F its float32 fraction.  Per cell,
 * moments (n_cells,27) f64 hold sum F_x^a F_y^b F_z^c (index 9a + 3b + c, a,b,c in 0..2).  S_ij =
 * sum_p phi_i(p) phi_j(p) and Phi_i = sum_p phi_i(p) (phi the trilinear weight, a polynomial in
 * F) are expanded from them in double.  Level l's cells sit on its grid (coarse node I at fine
 * node 2^l I); map (n^3) int32 = a cell's row in moments or -1; mask (n^3) u8 bit d (d = 4 dx +
 * 2 dy + dz) = cell node - d holds points.  g = alpha n_s / n = gamma h^2; level l uses
 * L_l - (gamma / 8^l) S_l, so its g is g / 2^l.  Boundary rules are those of the multigrid above.
 * casmvs_poisson_screen_keys: keys (n) int64 = flat splat cell, INT64_MAX when it leaves 0..N-2.
 * casmvs_poisson_screen_moments: the points order[cell_start[c] .. cell_start[c+1]) of each cell,
 *   summed in that order.
 * casmvs_poisson_screen_coarsen: parent cell (parent_keys, flat on the (n_child/2)^3 grid) = sum
 *   over its children m = 0..7 (x-major, child_map on the n_child^3 grid) of the child moments
 *   under F' = (m + F) / 2.
 * casmvs_poisson_screen_rhs: b_s = f32(b - gamma_t Phi) at interior nodes of level 0, 0 on the
 *   outer layer; *bb = sum of b_s^2.
 * casmvs_poisson_screen_stencil: for the nodes (n_nodes flat indices, mask != 0) of a level,
 *   the 27-point stencil of S (k = 9 (dx+1) + 3 (dy+1) + (dz+1)): sum over the cells d = 0..7
 *   around the node, then their corners, of S expanded from the moments in double; corners at
 *   index n drop.  stencil32 (n_nodes,27) f32 and/or stencil64 f64 (either may be NULL).
 *   srow (n^3) int32 = a node's row in the stencil arrays (read only where mask != 0).
 * casmvs_poisson_screen_residual: r = b_s - (sum of the 6 neighbours - 6 chi - g S chi) / h^2 in
 *   double on level 0 with the f64 stencil; *rr = sum of r^2 (before rounding).
 * casmvs_poisson_screen_mg_residual: out = r - (nbsum(e) - 6 e - g_l S e) / h^2 in f32 with the
 *   f32 stencil (S e summed in k order) at the level's interior nodes; 0 elsewhere.
 * casmvs_poisson_screen_smooth: `sweeps` 8-colour Gauss-Seidel sweeps, colour 4 (x&1) + 2 (y&1) +
 *   (z&1) in order 0..7, in f32: e = (nbsum(e) - h^2 r - g_l sum_{k != 13} S_k e_k) /
 *   (6 + g_l S_13), (nbsum(e) - h^2 r) / 6 where mask = 0; zero_first: start from e = 0 (in one
 *   block when n^3 <= 512). */
int casmvs_poisson_screen_keys(const float* points, int n, float h, int lo_x, int lo_y, int lo_z,
                               int N, long long* keys, void* stream);
int casmvs_poisson_screen_moments(const float* points, const int* order, const int* cell_start,
                                  int n_cells, float h, int lo_x, int lo_y, int lo_z,
                                  double* moments, void* stream);
int casmvs_poisson_screen_coarsen(const int* child_map, const double* child_moments, int n_child,
                                  const long long* parent_keys, int n_parents,
                                  double* parent_moments, void* stream);
int casmvs_poisson_screen_rhs(const float* b, const unsigned char* mask, const int* map,
                              const double* moments, int N, double gamma_t, float* b_s,
                              double* workspace, double* bb, void* stream);
int casmvs_poisson_screen_stencil(const long long* nodes, int n_nodes, const unsigned char* mask,
                                  const int* map, const double* moments, int n, float* stencil32,
                                  double* stencil64, void* stream);
int casmvs_poisson_screen_residual(const double* chi, const float* b_s, const unsigned char* mask,
                                   const int* srow, const double* stencil, int N, float h, double g,
                                   float* r, double* workspace, double* rr, void* stream);
int casmvs_poisson_screen_mg_residual(const float* e, const float* r, const unsigned char* mask,
                                      const int* srow, const float* stencil, int n, int level,
                                      float h, double g, float* out, void* stream);
int casmvs_poisson_screen_smooth(float* e, const float* r, const unsigned char* mask,
                                 const int* srow, const float* stencil, int n, int level, float h,
                                 double g, int sweeps, int zero_first, void* stream);

/* ---- quadric edge-collapse decimation (csrc/simplify.cu, casmvsnet_pl_b200/simplify.py) ----
 * A mesh is verts (V,3) f32, colours (V,3) u8, faces (F,3) int32, 3F < 2^31.  Every double
 * operation below is rounded to nearest in the order written, with no contraction; sums run in
 * a fixed order and the only atomics are integer ones, so results are bitwise reproducible.
 * Corner c = 3 f + k of face f sits at vertex faces[f][k] and owns the edge faces[f][k] --
 * faces[f][(k+1)%3].  Edges: edge_keys (E) int64 = (a << 32) | b, a < b, sorted and unique,
 * edge index = rank; corner_edge (3F) int32 = the edge a corner owns; edge_count (E) int32 =
 * faces on the edge (1 = boundary edge).  CSR: the corners at vertex v are
 * corners[off[v] .. off[v+1]) (int32), in increasing corner (so face) order.
 * Plane quadric of unit normal n^ through p0 with weight w: w [n^, -n^.p0][n^, -n^.p0]^T, as the
 * 10 unique entries (xx, xy, xz, xw, yy, yz, yw, zz, zw, ww), n^ = n / sqrt((nx nx + ny ny) + nz nz).
 * casmvs_simplify_clean: keep (F) u8 = 0 for a face with a repeated index or with
 *   n = (p1 - p0) x (p2 - p0) = 0 in double.
 * casmvs_simplify_frozen: frozen (V) u8 = 1 for a vertex with > 32 faces, on an edge of > 2
 *   faces, or whose link (an edge p-q per face (v, p, q)) is not connected (not one fan).
 * casmvs_simplify_face_quadrics: fq (F,10) f64, the plane quadric of n = (p1 - p0) x (p2 - p0)
 *   through p0 with weight |n| / 2.
 * casmvs_simplify_vertex_quadrics: Q (V,10) f64 = 0 + the fq of v's faces in face order + the
 *   quadrics of v's boundary edges in edge order: plane normal (pb - pa) x n_f of the edge's
 *   face f, through pa, weight 1000 |pb - pa|^2.
 * casmvs_simplify_edge_costs: deg (V) int32 = distinct neighbours, bnd (V) u8 = on a boundary
 *   edge (both zeroed and filled here); per edge, Q = Q_a + Q_b, A its upper-left 3x3:
 *   v = f32(Cramer's solution of A v = -Q[0:3,3]) when |det A| > 1e-12 max|A_ij|^3 and v is
 *   finite, else the first of a, b, f32((a + b) * 0.5) of least [v,1]^T Q [v,1];
 *   cost = f32(max(0, [v,1]^T Q [v,1])) (NaN stays NaN), newpos (E,3) f32 = v.
 *   valid0 (E) u8: cost finite, a and b not frozen, the common neighbours of a and b are
 *   exactly the opposite vertices of the faces on ab, not (a and b on the boundary and ab
 *   interior), deg a + deg b - 2 - common >= 3 (2 when a or b is on the boundary), deg c - 1 >= 3
 *   (2 on the boundary) for every opposite vertex c, faces(a) + faces(b) - faces(ab) <= 32, and
 *   every face around a or b without both has n_new . n_old > (0.2 |n_new|) |n_old| with the
 *   moved vertex at v.  key (E) int64 = (float bits of cost << 32) | e when valid0 and (unless
 *   !has_max_error) cost <= max_error, else INT64_MAX.
 * casmvs_simplify_select: m1 (V) = least key <= thr over the edges at v (INT64_MAX if none);
 *   m2 (V) = least m1 over v and the vertices of its faces; sel (E) u8 = key <= thr and
 *   key == m2[a] == m2[b].  No endpoint of one selected edge is in the 1-ring of another's.
 * casmvs_simplify_collapse: for the n edges idx (int64): a takes v = newpos[e], Q_a + Q_b and
 *   colour rint(c_a + t (c_b - c_a)), t = clamp(((v - a).(b - a)) / |b - a|^2, 0, 1) (0 when
 *   |b - a| = 0), remap[b] = a (remap otherwise as the caller set it).
 * casmvs_simplify_remap_faces: faces = map[faces] in place; keep (F) u8 = three distinct indices.
 * casmvs_simplify_mark_used: used (V) int32 = 1 for a vertex of a face, else 0 (zeroed here). */
int casmvs_simplify_clean(const float* verts, const int* faces, int F, unsigned char* keep,
                          void* stream);
int casmvs_simplify_frozen(const int* faces, int V, const int* off, const int* corners,
                           const int* corner_edge, const int* edge_count, unsigned char* frozen,
                           void* stream);
int casmvs_simplify_face_quadrics(const float* verts, const int* faces, int F, double* fq,
                                  void* stream);
int casmvs_simplify_vertex_quadrics(const float* verts, const int* faces, int V, const int* off,
                                    const int* corners, const int* corner_edge,
                                    const long long* edge_keys, const int* edge_count,
                                    const double* fq, double* Q, void* stream);
int casmvs_simplify_edge_costs(const float* verts, const double* Q, const int* faces, int V,
                               const int* off, const int* corners, const long long* edge_keys,
                               const int* edge_count, int E, const unsigned char* frozen,
                               int has_max_error, double max_error, int* deg, unsigned char* bnd,
                               float* newpos, float* cost, unsigned char* valid0, long long* key,
                               void* stream);
int casmvs_simplify_select(const long long* edge_keys, const long long* key, int E, long long thr,
                           const int* faces, int V, const int* off, const int* corners,
                           long long* m1, long long* m2, unsigned char* sel, void* stream);
int casmvs_simplify_collapse(const long long* edge_keys, const long long* idx, int n,
                             const float* newpos, float* verts, unsigned char* colours, double* Q,
                             int* remap, void* stream);
int casmvs_simplify_remap_faces(int* faces, int F, const int* map, unsigned char* keep,
                                void* stream);
int casmvs_simplify_mark_used(const int* faces, int F, int V, int* used, void* stream);

/* ---- uniform surface sampling (csrc/mesh_sample.cu, casmvsnet_pl_b200/mesh_sample.py) --------
 * Scores a mesh with the point-cloud scorers by sampling its surface.  A mesh is verts (V,3) f32
 * and faces (F,3) int32, 3F < 2^31.  Every double operation is rounded to nearest in the order
 * written, with no contraction, and no atomics are used, so results are bitwise reproducible.
 * For face f = (a, b, c) in its stored corner order, vertices read as double, with spacing s:
 *   L = the longest of |b - a|, |c - b|, |a - c|, |q - p| = sqrt((dx dx + dy dy) + dz dz),
 *   n = max(1, (int)min(ceil(L / s), 2^16)), count = (n + 1)(n + 2) / 2 samples;
 *   sample (i, j), i = 0..n, j = 0..n - i, has local index k = i (n + 1) - i (i - 1) / 2 + j and
 *   position f32((a + (i/n)(b - a)) + (j/n)(c - a)) per coordinate.
 * Output is face-major, then k; shared edges and vertices are sampled once per face.
 * casmvs_mesh_sample_count: n (F) int32 and count (F) int64 per face; spacing finite and > 0.
 * casmvs_mesh_sample_points: out (S,3) f32, S = sum of count < 2^31, given n and start (F) int64,
 *   the exclusive prefix sum of count.  One thread per sample. */
int casmvs_mesh_sample_count(const float* verts, const int* faces, int F, double spacing, int* n,
                             long long* count, void* stream);
int casmvs_mesh_sample_points(const float* verts, const int* faces, int F, const int* n,
                              const long long* start, long long S, float* out, void* stream);

/* ---- mesh cleaning (csrc/mesh_clean.cu, casmvsnet_pl_b200/mesh_clean.py) ----------------------
 * Drops small pieces and fills small holes.  A mesh, its edges and corners are as for
 * casmvs_simplify_* above; the faces here have passed casmvs_simplify_clean.  Every double
 * operation is rounded to nearest in the order written, with no contraction; the only atomics are
 * integer ones, so results are bitwise reproducible.
 * casmvs_mesh_clean_face_area: area (F) f64 = 0.5 sqrt(n.n), n = (p1 - p0) x (p2 - p0),
 *   n.n = (nx nx + ny ny) + nz nz.
 * casmvs_mesh_clean_sums: out[p] = 0 + value[order[start[p]]] + ... + value[order[start[p+1]-1]]
 *   summed left to right (order int64, or NULL for the identity).  A piece's area is the sum of
 *   its chunk sums, a chunk being up to 1024 of its faces in face order.
 * casmvs_mesh_clean_boundary: a boundary half-edge is corner c's directed edge a -> b with
 *   edge_count = 1.  out_deg / in_deg (V) int32 count them at a and b; next (V) int32 = b and
 *   next_face (V) int32 = c / 3 where a has out_deg = in_deg = 1, else -1 (all set here).
 * casmvs_mesh_clean_loop_sizes: with comp (V) the least vertex of each component of the graph
 *   v -- next[v] over the vertices with next >= 0 (casmvs_texture_charts): size (V) int32 counts
 *   the vertices with next >= 0 per root, open (V) u8 = 1 at a root whose component holds a v with
 *   next[next[v]] < 0 (a path, not a loop); both zeroed here.
 * casmvs_mesh_clean_fill: one loop per owner[L] (its least vertex) of size[L] = n in 3..max_size
 *   <= 128 edges; position i is next^i(owner).  cost(i, i+1) = 0; for j - i >= 2,
 *   cost(i, j) = min over i < k < j of (cost(i, k) + cost(k, j)) + 0.5 sqrt(m.m),
 *   m = (p_k - p_i) x (p_j - p_i), least k on ties, skipping k with m = 0, and +inf when (i, j) is
 *   not 0 -- n-1 and the edge vid_i -- vid_j is in edge_keys (E sorted int64, binary search) or
 *   when no k is admissible.  area[L] f64 = cost(0, n-1); status[L] u8 = 2 when it is +inf, else
 *   1 when area <= 0.1 x piece_area[next_face[owner]] (piece_area per face), else 3.
 *   tris (sum (n - 2), 3) int32 from row tri_off[L] (int64): pre-order from (0, n-1), (i, j)
 *   emitting (vid_j, vid_k, vid_i) with its split k, then (i, k), then (k, j); -1 when status 2. */
int casmvs_mesh_clean_face_area(const float* verts, const int* faces, int F, double* area,
                                void* stream);
int casmvs_mesh_clean_sums(const double* value, const long long* order, const long long* start,
                           int n, double* out, void* stream);
int casmvs_mesh_clean_boundary(const int* faces, int F, const int* corner_edge,
                               const int* edge_count, int V, int* out_deg, int* in_deg, int* next,
                               int* next_face, void* stream);
int casmvs_mesh_clean_loop_sizes(const int* next, const int* comp, int V, int* size,
                                 unsigned char* open, void* stream);
int casmvs_mesh_clean_fill(const float* verts, const int* next, const int* next_face,
                           const int* owner, const int* size, int n_loops, int max_size,
                           const long long* tri_off, const long long* edge_keys, int E,
                           const double* piece_area, unsigned char* status, double* area, int* tris,
                           void* stream);

/* ---- headless rendering of clouds and meshes (casmvsnet_pl_b200/render.py) -----------------
 * P is a HOST array of 16 floats, row-major, world -> pixel (rows 0..2 used): every float
 * operation below is rounded to nearest, no contraction, in the order written.
 *   w = ((P20 X + P21 Y) + P22 Z) + P23, likewise x (row 0) and y (row 1); u = x / w, v = y / w.
 * A vertex or point is drawn only when X, Y, Z, w, u, v are finite and w > 0; there is no near-
 * plane clipping, so a triangle with one vertex at w <= 0 is skipped whole.  Pixel (px, py) has
 * its centre at the integers (px, py), row-major.  zbuf (H*W) u64 is caller-provided and filled
 * here: each covered pixel takes atomicMin of key = (float bits of w) << 32 | primitive index, so
 * the nearest primitive wins and an exact depth tie goes to the lower index (deterministic).
 * image (H,W,3) u8 gets the winner's colour or the background (128, 128, 255); depth (H,W) f32
 * the winner's w, 0 where nothing is drawn.  1 <= W, H <= 16384.
 * casmvs_render_points_fwd: xyz (n,3) f32, rgb (n,3) u8, n < 2^32.  A point of size s (1..64)
 *   covers the pixel centres in [u - s/2, u + s/2) x [v - s/2, v + s/2): px from
 *   ceil(u - s/2) to ceil(u + s/2) - 1, likewise py.
 * casmvs_render_mesh_fwd: verts (n_vertices,3) f32, colours (n_vertices,3) u8, faces (n_faces,3)
 *   int32; eye a HOST array of 3 floats (the camera centre).  Both windings are drawn.  Face t is
 *   skipped unless its area a = e(u0,v0, u1,v1, u2,v2) != 0, with
 *     e(ax,ay, bx,by, px,py) = (bx - ax)(py - ay) - (by - ay)(px - ax).
 *   It covers pixel (px, py) of its box [ceil(min u), floor(max u)] x [ceil(min v), floor(max v)]
 *   when e0 = e(1,2,p), e1 = e(2,0,p), e2 = e(0,1,p) are all >= 0 or all <= 0; then
 *     q_k = e_k / w_k, den = (q0 + q1) + q2, depth = ((e0 + e1) + e2) / den (drawn if > 0, finite)
 *     colour_c = floor((((q0 c0 + q1 c1) + q2 c2) / den) * shade + 0.5), clamped to 0..255,
 *     shade = 0.3 + 0.7 min(1, |n.d| / (sqrt(n.n) sqrt(d.d))) (0.3 when the divisor is 0),
 *     n = (x1 - x0) x (x2 - x0), d = ((x0 + x1) + x2) / 3 - eye, dots summed ((a0 + a1) + a2).
 *   A face index outside [0, n_vertices) is caught on the device: nothing is read through it and
 *   the call fails.  The call synchronises `stream` once, to read that flag.  Boxes up to 8x8
 *   pixels are rasterised by one thread per face, larger ones by a CTA each.
 * casmvs_render_mesh_workspace_bytes: the workspace (4-byte aligned) for n_faces faces. */
int casmvs_render_points_fwd(const float* xyz, const unsigned char* rgb, long long n, const float* P,
                             int W, int H, int point_size, unsigned long long* zbuf,
                             unsigned char* image, float* depth, void* stream);
size_t casmvs_render_mesh_workspace_bytes(int n_faces);
int casmvs_render_mesh_fwd(const float* verts, const unsigned char* colours, int n_vertices,
                           const int* faces, int n_faces, const float* P, const float* eye, int W,
                           int H, unsigned long long* zbuf, void* workspace,
                           size_t workspace_bytes, unsigned char* image, float* depth,
                           void* stream);

/* ---- mesh texturing from the views (csrc/texture.cu, casmvsnet_pl_b200/texture.py) -----------
 * casmvs_render_mesh_keys: the raster pass of casmvs_render_mesh_fwd alone (same arguments, same
 *   zbuf bits): the view's visibility buffer.
 * casmvs_render_textured_mesh_fwd: the raster pass, then per covered pixel the winner t's UV
 *   tu = (((q0 U0 + q1 U1) + q2 U2) / den), likewise tv, from uv (n_faces,3,2) f32 (corner k of
 *   face t at uv[t][k]); x = tu S - 0.5, y = (1 - tv) S - 0.5, each clamped to [-1, S];
 *   i = floor, a = x - floor(x) (likewise y); the four texels (i, i + 1) x (j, j + 1) clamped to
 *   0..S-1 of page[t] in atlas (n_pages,S,S,3) u8 (row j, column i) give
 *   c = floor(((1 - ay) ((1 - ax) c00 + ax c10) + ay ((1 - ax) c01 + ax c11)) + 0.5), clamped to
 *   0..255, per channel.  Unshaded.  depth as render_mesh_fwd.
 * The texturing rule.  Constants: K = 4 candidates, PAD = 2, MIN_COS = 0.1, DEPTH_TOL = 0.01
 * (the float 1.01f below), at most 8 views per scores call.  Views are P (4,4) f32 row-major
 * world -> pixel and the eye (3) f64, the camera centre solved from P in double.
 * casmvs_texture_scores: for n_views views of one batch (HOST arrays: P n*16 f32, eye n*3 f64,
 *   wh n*2 int32, view_index n int32, zbufs n DEVICE key buffers of casmvs_render_mesh_keys),
 *   one thread per face f of corners x0, x1, x2 (f32): n = (x1 - x0) x (x2 - x0) and the centroid
 *   c = ((x0 + x1) + x2) / 3 in double, c' the same in float32.  f is a candidate in view j when
 *   n.n > 0; x0, x1, x2 and c' project (render_mesh_fwd's projection); each vertex has
 *   PAD <= u <= W-1-PAD and PAD <= v <= H-1-PAD; |n.d| >= 0.1 (sqrt(n.n) sqrt(d.d)), d = c - eye,
 *   dots ((a0 b0 + a1 b1) + a2 b2); and each of the four samples has a non-empty key at pixel
 *   (rint(u), rint(v)) with w <= f32(depth * 1.01f).  Score = f32(0.5 |(u1-u0)(v2-v0) -
 *   (v1-v0)(u2-u0)|) in double.  cand_score (F,4) f32 and cand_view (F,4) int32 (-1 = empty, the
 *   caller's initial state) keep the best 4 by (score desc, view asc) across calls made in view
 *   order.
 * casmvs_texture_smooth: one Jacobi round over label_in -> label_out (F) int32.  nbr (F,3) int32
 *   is the face across the edge of corner k (faces[f][k] -- faces[f][(k+1)%3]) when exactly two
 *   distinct faces share it, else -1.  f takes L when >= 2 of its nbr held L and L is one of its
 *   candidates with score >= f32(0.5 * best score); otherwise it keeps label_in[f].
 * casmvs_texture_charts: comp (F) int32 = the least face index of f's component: faces joined
 *   across nbr edges with equal labels >= 0 (a face of label -1 is alone).  atomicMin hooking and
 *   pointer jumping, repeated until a hook round changes nothing (flag: 4 device bytes; *rounds,
 *   HOST, the hook rounds).  Synchronises stream once per round.
 * casmvs_texture_rects: rect (F,4) int32, filled here: for a root r, (min x0, min y0, max x1,
 *   max y1) over its faces of label L >= 0 with x0 = floor(min u) - PAD, x1 = ceil(max u) + PAD
 *   (v likewise) of the face's corners projected by Ps[L] (Ps (n_views,16) f32, DEVICE);
 *   (INT_MAX, INT_MAX, INT_MIN, INT_MIN) elsewhere.
 * charts (n_charts,9) int32 rows: root face, view (-1 = flat), x0, y0, x1, y1, page, ox, oy.
 * casmvs_texture_fill: atlas (pages,S,S,3) u8, zeroed by the caller; a view chart's
 *   (x1-x0+1) x (y1-y0+1) texels at (ox, oy) of its page are the bytes of its rectangle in
 *   images[view] (DEVICE array of (H,W,3) u8 device pointers, wh (n_views,2) int32 DEVICE); a flat
 *   chart's 4 x 4 texels are the root face's vertex colours' mean, (sum + 1) / 3 per channel
 *   (round half to even, as a third is never a half).
 * casmvs_texture_uvs: slot (F) int32 = the chart row of f.  page[f] = its page; corner k of a view
 *   chart's face: (u, v) projected by Ps[label], uv = f32((((u - x0) + ox) + 0.5) / S),
 *   f32(1 - (((v - y0) + oy) + 0.5) / S) in double; of a flat face: the texel centres
 *   (1.5, 1.5), (2.5, 1.5), (1.5, 2.5) of its square, f32((o + c) / S) and f32(1 - (o + c) / S). */
int casmvs_render_mesh_keys(const float* verts, int n_vertices, const int* faces, int n_faces,
                            const float* P, int W, int H, unsigned long long* zbuf,
                            void* workspace, size_t workspace_bytes, void* stream);
int casmvs_render_textured_mesh_fwd(const float* verts, int n_vertices, const int* faces,
                                    int n_faces, const float* uv, const int* page,
                                    const unsigned char* atlas, int n_pages, int S, const float* P,
                                    int W, int H, unsigned long long* zbuf, void* workspace,
                                    size_t workspace_bytes, unsigned char* image, float* depth,
                                    void* stream);
int casmvs_texture_scores(const float* verts, const int* faces, int F, int n_views, const float* P,
                          const double* eye, const int* wh, const int* view_index,
                          unsigned long long* const* zbufs, float* cand_score, int* cand_view,
                          void* stream);
int casmvs_texture_smooth(const int* nbr, const float* cand_score, const int* cand_view, int F,
                          const int* label_in, int* label_out, void* stream);
int casmvs_texture_charts(const int* nbr, const int* label, int F, int* comp, unsigned* flag,
                          int* rounds, void* stream);
int casmvs_texture_rects(const float* verts, const int* faces, int F, const int* label,
                         const int* comp, const float* Ps, int* rect, void* stream);
int casmvs_texture_fill(const int* charts, int n_charts, const unsigned long long* images,
                        const int* wh, const unsigned char* colours, const int* faces, int S,
                        unsigned char* atlas, void* stream);
int casmvs_texture_uvs(const float* verts, const int* faces, int F, const int* label,
                       const int* slot, const int* charts, const float* Ps, int S, float* uv,
                       int* page, void* stream);

/* ---- seam levelling of a textured mesh (csrc/texture_level.cu, casmvsnet_pl_b200/texture.py) --
 * Waechter et al. 2014's global colour adjustment, run on texture_mesh's labels, slot, charts,
 * nbr and atlas.  Constants: SEAM_SAMPLES = 8, SMOOTH_WEIGHT = 10, EPS = 1e-4, REACH = 1.5 texels.
 * Every double operation below is rounded as written (no contraction), left to right.
 * casmvs_texture_level_keys: keys (3F) int64 = (slot[f] << 32) | faces[f][k] for a face of label
 *   >= 0, else -1.  The unknowns are the distinct keys >= 0 in ascending order (one RGB offset g
 *   per (chart, vertex) pair), n of them, sorted by the caller.
 * casmvs_texture_level_corners: corner (3F) int32 = the index of keys[i] among the n unknowns
 *   (-1 for a flat face).
 * casmvs_texture_level_edges: per corner c = 3f + k, the edge faces[f][k] -- faces[f][(k+1)%3]:
 *   smooth_key[c] = (min << 32) | max of its two corners' unknowns when label[f] >= 0 and they
 *   differ, else -1 (the caller keeps the distinct keys: the smoothing edges);
 *   rec_key[2c + e] (e = 0 for the corner-k endpoint, 1 for the other) = (a << 32) | b, a < b the
 *   endpoint's unknowns in the two charts, when the edge is a seam seen from its lower face:
 *   g = nbr[f][k] >= 0, f < g, label[f] >= 0, label[g] >= 0, slot[f] != slot[g]; else -1.  A seam
 *   pair is a distinct such key; the caller keeps the records rec_sub = 2c + e with a key,
 *   stably sorted by key.
 * casmvs_texture_level_samples: rec (R,6) f64 per record: for s = 0..7, t = s / 8, the point
 *   X = x0 + t (x1 - x0) per coordinate in double (x0 the record's endpoint, x1 the edge's other
 *   end, f32 vertices), projected by Ps[view] as u = (((P0 X + P1 Y) + P2 Z) + P3) / w (w and v
 *   likewise, P widened to double), clamped to [0, W-1] x [0, H-1]; a = u - floor(u), the taps
 *   (floor, floor + 1 clamped to W-1) of images[view] (pixel centres at integer coordinates)
 *   c = (1 - ay) ((1 - ax) c00 + ax c10) + ay ((1 - ax) c01 + ax c11); acc += (1 - t) c.
 *   Columns 0..2 in the view of the lower chart (the chart of unknown a), 3..5 in the upper's.
 * casmvs_texture_level_pairs: fpair (P,6) f64: per pair, num = sum of its records' rec and
 *   den = sum of W = sum_s (1 - s / 8), both from 0 in record order; f = num / den, f_a in
 *   columns 0..2, f_b in 3..5.
 * casmvs_texture_level_system: ekey (nnz) int64 ascending = (row << 32) | col of every entry:
 *   both orders of each seam pair and smoothing edge, and (a, a) per unknown; etype (nnz) int32
 *   = the seam pair's index, -2 for a smoothing edge, -1 for the diagonal.  Writes rowptr (n+1),
 *   col (nnz) int32 and val (nnz), diag (n), rhs (n,3) f64, one thread per row in column order:
 *   off-diagonal -1 (seam) or -10 (smoothing), s = their sum from 0, diagonal -s + EPS;
 *   rhs[a] += f_b - f_a over the row's seam pairs with a the row's unknown (f_a - f_b when it is
 *   b), from 0.  This is A g = rhs for the minimum of sum_pairs (f_a + g_a - f_b - g_b)^2
 *   + SMOOTH_WEIGHT sum_edges (g_a - g_b)^2 + EPS sum g^2.
 * casmvs_texture_level_cg: Jacobi-preconditioned CG from x = 0 on the three columns of rhs at
 *   once (x (n,3) f64), until every column has ||r|| / ||b|| <= tol (0 when b = 0) or after
 *   max_iters iterations.  Dot products are per-thread sums in grid-stride order, a fixed
 *   256-wide tree per block and one block over the block partials, over min(1024, ceil(n/256))
 *   blocks.  alpha = rz / pq (0 unless pq > 0), beta = rz' / rz (0 unless rz > 0).  The host
 *   reads the done flag every check_every iterations; iterations after convergence are no-ops,
 *   so *iters does not depend on check_every.  HOST outputs: *iters, ratios[3], *converged.
 *   workspace: casmvs_texture_level_cg_workspace_bytes(n).
 * casmvs_texture_level_owners: owner (pages,S,S) u64, all ~0 from the caller.  One warp per face
 *   of label L >= 0: its corners projected by Ps[L] (the UVs' f32 projection) widened to double;
 *   for every integer view pixel p = (x, y) of its chart's rectangle within REACH of the
 *   triangle's bounding box, the nearest point of the triangle: inside (area = (u1-u0)(v2-v0) -
 *   (v1-v0)(u2-u0) != 0 and l_k = ((u_{k+1}-x)(v_{k+2}-y) - (v_{k+1}-y)(u_{k+2}-x)) / area >= 0
 *   for all k) -> distance 0, barycentrics l; else the edge k -> k+1 of least squared distance
 *   (ties to the lower k), t = clamp(((x-u_k) du + (y-v_k) dv) / (du du + dv dv), 0, 1) (0 for a
 *   zero-length edge), e = p - (P_k + t d), d2 = ex ex + ey ey, distance sqrt(d2), barycentrics
 *   1 - t at k and t at k+1.  When distance <= REACH, atomicMin(owner[page][oy + y - y0][ox + x -
 *   x0], (f32(distance) bits << 32) | f).
 * casmvs_texture_level_apply: per atlas texel (64-bit index over n_texels = pages S S) with an
 *   owner f: the nearest point's barycentrics l of its view pixel as above, offset
 *   o = ((l0 g[c0] + l1 g[c1]) + l2 g[c2]) per channel (c_k = corner[3f + k], g (n,3) f64), and
 *   the byte becomes min(max(rint(byte + o), 0), 255) (rint: half to even).  Texels without an
 *   owner, flat charts and unused texels are untouched. */
int casmvs_texture_level_keys(const int* faces, int F, const int* label, const int* slot,
                              long long* keys, void* stream);
int casmvs_texture_level_corners(const long long* keys, int F, const long long* unknowns, int n,
                                 int* corner, void* stream);
int casmvs_texture_level_edges(const int* nbr, const int* faces, int F, const int* label,
                               const int* slot, const int* corner, long long* rec_key,
                               long long* smooth_key, void* stream);
int casmvs_texture_level_samples(const float* verts, const int* faces, const int* label,
                                 const int* slot, const int* nbr, const long long* rec_sub, int R,
                                 const float* Ps, const unsigned long long* images, const int* wh,
                                 double* rec, void* stream);
int casmvs_texture_level_pairs(const double* rec, const long long* seg, int P, double* fpair,
                               void* stream);
int casmvs_texture_level_system(const long long* ekey, const int* etype, long long nnz, int n,
                                const double* fpair, int* rowptr, int* col, double* val,
                                double* diag, double* rhs, void* stream);
size_t casmvs_texture_level_cg_workspace_bytes(int n);
int casmvs_texture_level_cg(const int* rowptr, const int* col, const double* val,
                            const double* diag, const double* rhs, int n, double* x,
                            void* workspace, size_t workspace_bytes, int max_iters, double tol,
                            int check_every, int* iters, double* ratios, int* converged,
                            void* stream);
int casmvs_texture_level_owners(const float* verts, const int* faces, int F, const int* label,
                                const int* slot, const int* charts, const float* Ps, int S,
                                unsigned long long* owner, void* stream);
int casmvs_texture_level_apply(const unsigned long long* owner, long long n_texels,
                               const float* verts, const int* faces, const int* label,
                               const int* slot, const int* charts, const float* Ps, int S,
                               const int* corner, const double* g, unsigned char* atlas,
                               void* stream);

/* ---- mesh refinement against the views (csrc/refine.cu, casmvsnet_pl_b200/refine.py) ----------
 * Moves vertex positions only.  Constants: R = 2 (a 5 x 5 patch), K = 4, STEP = 1, SPACING = 4,
 * S_MAX = 4, VAR_MIN = 1e-4, MIN_GAIN = 5e-4, MIN_SCORE = 0.3, lambda = 1; PAD = 2, MIN_COS = 0.1 and DEPTH_TOL = 0.01 as in
 * texturing; at most 8 views per visibility call.  The caller runs, per iteration it = 0 .. T-1:
 * normals, the key buffers of the current mesh (casmvs_render_mesh_keys) and visibility one batch
 * at a time, selection, the sweep, J = 4 smoothing rounds from d = d0, and apply.  Each vertex is
 * one thread; sums run in the order stated; there are no atomics.
 * casmvs_refine_grey: grey (n) f64 = ((0.299 R + 0.587 G) + 0.114 B) / 255 of rgb (n,3) u8,
 *   each operation rounded.
 * casmvs_refine_normals: normal (V,3) f64 = s / |s|, s the sum from 0 over vf_face[vf_ptr[v] ..
 *   vf_ptr[v+1]) (the faces of v, ascending) of (x1 - x0) x (x2 - x0) in double, each operation
 *   rounded as written ((a1 b2 - a2 b1) etc., |s| = sqrt((s0 s0 + s1 s1) + s2 s2)); 0 when |s| = 0.
 * casmvs_refine_visibility: for the views of one batch (HOST arrays as casmvs_texture_scores':
 *   P n*16 f32, eye n*3 f64, wh n*2, view_index n, zbufs n DEVICE key buffers), sets bit
 *   view_index[j] of vertex v in vis (V, words) u32 (zeroed by the caller before the first batch)
 *   when v projects (render_mesh_fwd's projection) with PAD <= u <= W-1-PAD, PAD <= v <= H-1-PAD,
 *   the key at (rint(u), rint(v)) is not empty and w <= f32(depth * 1.01f), and
 *   |n.d| >= 0.1 sqrt(d.d), d = eye - v, dots ((a0 b0 + a1 b1) + a2 b2).
 * casmvs_refine_select: ref (V) int32 = the visible view of largest |n.d| / sqrt(d.d) (ties to the
 *   lower index; eyes (n_views,3) f64 DEVICE); src (V,4) int32 = the reference's sources
 *   src_ids[src_ptr[ref] .. src_ptr[ref+1]) (DEVICE CSR over the views) in which v is visible, in
 *   that order, at most 4, -1 after the last.  ref = -1 without a reference or a source.
 * casmvs_refine_sweep: per vertex with ref >= 0: rho, the tangent frame, the candidates at
 *   delta_k = k rho 2^-iteration and the ZNCC scores S_k of csrc/refine.cu's rule, step 4, in
 *   double; Ps (n,16) f32 and Pinv (n,16) f64 (inv of P in double) DEVICE; grey DEVICE array of
 *   (H,W) f64 device pointers (casmvs_refine_grey), wh (n,2) int32 DEVICE.  Outputs (V): rho,
 *   best = S_k* (NaN without a valid k), kstar (-1000 without one), d (step 5's d, 0 unless
 *   confident), conf (c); sk (V,9) f64 (NaN where k is invalid) only when not NULL.
 * casmvs_refine_smooth: one Jacobi round d_out = (conf d0 + sum d_in[nb]) / (conf + |nb|), the sum
 *   from 0 over nb_ids[nb_ptr[v] .. nb_ptr[v+1]) (the one-ring, ascending); 0 when the divisor is 0.
 * casmvs_refine_apply: verts_out = f32(verts_in + d normal) per coordinate, in double. */
int casmvs_refine_grey(const unsigned char* rgb, long long n_pixels, double* grey, void* stream);
int casmvs_refine_normals(const float* verts, int V, const int* faces, const int* vf_ptr,
                          const int* vf_face, double* normal, void* stream);
int casmvs_refine_visibility(const float* verts, const double* normal, int V, int n_views,
                             const float* P, const double* eye, const int* wh,
                             const int* view_index, unsigned long long* const* zbufs,
                             unsigned* vis, int words, void* stream);
int casmvs_refine_select(const float* verts, const double* normal, int V, const unsigned* vis,
                         int words, int n_views, const double* eyes, const int* src_ptr,
                         const int* src_ids, int* ref, int* src, void* stream);
int casmvs_refine_sweep(const float* verts, const double* normal, int V, const int* ref,
                        const int* src, const float* Ps, const double* Pinv,
                        const unsigned long long* grey, const int* wh, int iteration, double* rho,
                        double* best, int* kstar, double* d, double* conf, double* sk,
                        void* stream);
int casmvs_refine_smooth(const int* nb_ptr, const int* nb_ids, int V, const double* d0,
                         const double* conf, const double* d_in, double* d_out, void* stream);
int casmvs_refine_apply(const float* verts_in, const double* normal, const double* d, int V,
                        float* verts_out, void* stream);

/* ---- training panels (csrc/visual.cu; utils/visualization.py, train.py:107-114) ---------
 * The original's TensorBoard image strip as uint8 (H, n*W, 3), n = the number of non-NULL panel
 * inputs, panels left to right in the order img, depth_gt, depth_pred, conf:
 *   img (3,H,W) f32, normalised as the data readers leave it -> un-normalised RGB;
 *   depth_gt (H,W) f32 -> visualize_depth(depth_gt);
 *   depth_pred (H,W) f32 -> visualize_depth(depth_pred * mask);
 *   conf (H,W) f32 -> visualize_prob(conf * mask).
 * mask (H,W) u8 (nonzero = valid) may be NULL: all valid.  The bytes equal the original's chain
 * (cv2 colour maps with blue and red swapped, numpy's wrapping float -> uint8 cast); a depth map
 * with no positive value is drawn in the colour of grey level 0, where the original raises.
 * workspace: CASMVS_VISUAL_WORKSPACE_BYTES, 16-byte aligned, needed with a depth panel; nothing
 * is read from it before the call writes it.  H * W < 2^31. */
#define CASMVS_VISUAL_WORKSPACE_BYTES 4096
int casmvs_visual_panels(const float* img, const float* depth_gt, const float* depth_pred,
                         const float* conf, const unsigned char* mask, int H, int W,
                         unsigned char* out, void* workspace, void* stream);

/* ---- layout helpers ------------------------------------------------------ */
/* (N,C,S) -> (N,S,C) and back, S = product of spatial dims. */
int casmvs_nchw_to_nhwc(const float* in, float* out, int N, int C, size_t S, void* stream);
int casmvs_nhwc_to_nchw(const float* in, float* out, int N, int C, size_t S, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CASMVS_H_ */
