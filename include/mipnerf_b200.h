/* mipnerf_b200.h — C ABI of libmipnerf_b200.so: the H100 (sm_90a) Mip-NeRF per-ray hot path.
 *
 * The reference (hjxwhy/mipnerf_pl) has no FFI layer: its boundary for this path is the Python
 * call surface `MipNerf.forward` (models/mip_nerf.py:172-248) and the free functions it reaches in
 * models/mip.py.  Each entry point below names the reference function it replaces.  The host-side
 * mirror that binds these symbols (ctypes) is mipnerf_pl_b200/_cabi.py; INTEGRATION.md shows the
 * stub a maintainer of the reference would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to row-major fp32 unless stated otherwise; the library never
 *     allocates or frees device memory and keeps no state besides the thread-local error string;
 *   - `stream` is a cudaStream_t passed as void*; all calls are asynchronous on it (no sync inside);
 *   - return value: 0 on success, negative MIPNERF_B200_E* on failure (`mipnerf_b200_last_error()`
 *     gives the text).  There is no CPU fallback anywhere behind this ABI.
 */
#ifndef MIPNERF_B200_H_
#define MIPNERF_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MIPNERF_B200_ABI_VERSION 4

#define MIPNERF_B200_OK 0
#define MIPNERF_B200_EINVAL (-1)       /* bad argument (NULL pointer, negative size, ...)            */
#define MIPNERF_B200_EUNSUPPORTED (-2) /* config outside what the kernels implement                  */
#define MIPNERF_B200_ECUDA (-3)        /* a CUDA runtime call or launch failed                       */
#define MIPNERF_B200_EWORKSPACE (-4)   /* workspace smaller than mipnerf_b200_workspace_bytes()      */

/* Arithmetic the MLP contraction runs in (everything else on the path is always fp32).
 * FP32 takes any config check_config accepts.  The tensor-core precisions take the reference's shipped architecture:
 * 8x256 trunk with the skip after layer 4, one 128-wide view layer, num_samples = 128 or 256, use_viewdirs,
 * min_deg_point = 0, max_deg_point 1..16 and deg_view 1..4 (narrower encodings are zero-padded into the operand image
 * by mipnerf_b200_pack_weights; the image does not depend on num_samples); the tensor-core TRAINING step and
 * mipnerf_b200_mlp_forward need max_deg_point = 16 and deg_view = 4, and mipnerf_b200_mlp_forward 128 samples per ray.
 * Anything else answers MIPNERF_B200_EUNSUPPORTED (mipnerf_b200_packed_weights_bytes() == 0). */
#define MIPNERF_B200_FP32 0 /* CUDA-core FFMA, fp32 operands: the 1e-4 parity mode                   */
#define MIPNERF_B200_BF16 1 /* wgmma, bf16 operands, fp32 accumulate                                */
#define MIPNERF_B200_FP16 2 /* wgmma, fp16 operands, fp32 accumulate                                */
/* Split-operand tensor-core modes: every GEMM operand x is carried as hi = fl16(x), lo = fl16(x - hi) and each
 * K step issues hi.hi + lo.hi + hi.lo into the same fp32 accumulator (3x the MMAs).  FP16X3 keeps 22
 * significant operand bits (|x| < 65504) and is the tensor-core mode that meets the reference's fp32 result
 * to 1e-4 (models/mip_nerf.py:94-110 computes every nn.Linear in fp32); BF16X3 keeps 16 bits with fp32's range. */
#define MIPNERF_B200_FP16X3 3
#define MIPNERF_B200_BF16X3 4

/* One torch.nn.Linear: weight [out_features, in_features] row-major, bias [out_features]. */
typedef struct mipnerf_b200_linear {
  const float* weight;
  const float* bias;
  int32_t in_features;
  int32_t out_features;
} mipnerf_b200_linear;

/* Constructor arguments of MipNerf that change the arithmetic (models/mip_nerf.py:117-141). */
typedef struct mipnerf_b200_config {
  int32_t num_samples; /* per level; CUDA path needs num_samples % 32 == 0 and <= 256               */
  int32_t num_levels;
  int32_t min_deg_point, max_deg_point, deg_view;
  int32_t use_viewdirs, disparity, disable_integration;
  float resample_padding, density_bias, rgb_padding;
  int32_t net_depth, net_width, net_depth_condition, net_width_condition, skip_index;
  int32_t num_rgb_channels, num_density_channels; /* must be 3 and 1                                */
  float density_noise; /* std of the Gaussian noise added to raw density when randomized (models/mip_nerf.py:232-233) */
} mipnerf_b200_config;

/* MLP parameters in state_dict order (models/mip_nerf.py:19-73):
 * layers.0 .. layers.{net_depth-1}, density_layer, extra_layer, view_layers.0 .. , color_layer.
 * `packed` is the optional tensor-core operand image written by mipnerf_b200_pack_weights. */
typedef struct mipnerf_b200_weights {
  const mipnerf_b200_linear* linears;
  int32_t num_linears;
  int32_t packed_precision; /* MIPNERF_B200_BF16/FP16 the image was packed for, or -1              */
  const void* packed;
  size_t packed_bytes;
} mipnerf_b200_weights;

/* Rays namedtuple fields used by forward (datasets/datasets.py:13-16; lossmult is not read). */
typedef struct mipnerf_b200_rays {
  const float* origins;    /* [B,3] */
  const float* directions; /* [B,3] not normalised */
  const float* viewdirs;   /* [B,3] */
  const float* radii;      /* [B,1] */
  const float* near;       /* [B,1] */
  const float* far;        /* [B,1] */
  int64_t num_rays;
} mipnerf_b200_rays;

/* One element of the list MipNerf.forward returns (models/mip_nerf.py:246). */
typedef struct mipnerf_b200_level_out {
  float* comp_rgb;  /* [B,3]            */
  float* distance;  /* [B]              */
  float* acc;       /* [B]              */
  float* weights;   /* [B,N]   nullable */
  float* t_samples; /* [B,N+1] nullable */
  int64_t* inds;    /* [B,N+1] nullable; searchsorted indices of the resampler (levels >= 1)       */
  /* INPUT, nullable: [B,N] standard-normal draws replacing torch.randn of models/mip_nerf.py:233 for this level.
   * Read only when randomized != 0 and cfg->density_noise > 0; required then by the entry points that take injected
   * noise (t_rand / u_jitter), ignored by the _rng entry points (in-kernel Philox + Box-Muller, stream 32 + level). */
  const float* density_normal;
} mipnerf_b200_level_out;

/* In-kernel random numbers for randomized=True: Philox4x32-10 keyed by `seed`; the draw of (ray, index, stream) is a
 * pure function of (seed, offset, ray's position in the call), so results do not depend on chunking.  Advance `offset`
 * by one per call for fresh noise (the role of torch's generator offset). */
typedef struct mipnerf_b200_rng {
  uint64_t seed;
  uint64_t offset;
} mipnerf_b200_rng;

const char* mipnerf_b200_last_error(void);
int mipnerf_b200_abi_version(void);

/* Bytes of scratch `mipnerf_b200_forward` / `mipnerf_b200_mlp_forward` need for `num_rays` rays. */
size_t mipnerf_b200_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_rays, int precision);

/* Size of / builder for the tensor-core operand image of the MLP weights (device -> device). */
size_t mipnerf_b200_packed_weights_bytes(const mipnerf_b200_config* cfg, int precision);
int mipnerf_b200_pack_weights(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                              int precision, void* packed_out, size_t packed_bytes, void* stream);

/* MipNerf.forward (models/mip_nerf.py:172-248).  `t_rand` [B,N+1] in [0,1) and `u_jitter`
 * [B,N+1] in [0, 1/(N+1)-eps) replace torch.rand / uniform_ (models/mip.py:159, :201-202) when
 * `randomized` != 0 (both required then).  `outs` has cfg->num_levels entries. */
int mipnerf_b200_forward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                         const mipnerf_b200_rays* rays, int randomized, const float* t_rand,
                         const float* u_jitter, int white_bkgd, int precision,
                         mipnerf_b200_level_out* outs, void* workspace, size_t workspace_bytes,
                         void* stream);

/* Same, drawing the uniforms of randomized mode INSIDE the kernels that consume them (no torch.rand launch, no
 * [B,N+1] arrays in HBM): stream 0 = the stratified draws of sample_along_rays (models/mip.py:159), stream 1+l =
 * the inverse-CDF jitter of level l (models/mip.py:201-202, scaled to [0, 1/(N+1) - eps)). */
int mipnerf_b200_forward_rng(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                             const mipnerf_b200_rays* rays, const mipnerf_b200_rng* rng, int white_bkgd,
                             int precision, mipnerf_b200_level_out* outs, void* workspace,
                             size_t workspace_bytes, void* stream);

/* Levels 1 .. num_levels - 1 of mipnerf_b200_forward's loop, run exactly as that loop runs them, with the caller's
 * fenceposts t_prev [B,N+1] and weights w_prev [B,N] in place of level 0's outputs (e.g. mipnerf_b200_grid_proposal's
 * weights at sample_along_rays' fenceposts: level 0's MLP is not run).  `outs` has cfg->num_levels - 1 entries, outs[k]
 * for level k + 1.  Draws as the forward's: `u_jitter` (required when randomized) is level l's inverse-CDF jitter for
 * every level, outs[k].density_normal the density noise of level k + 1; the _rng form draws stream 1 + l (jitter) and
 * 32 + l (density noise) of `rng`.  So with t_prev / w_prev = a forward's outs[0].t_samples / weights, every output
 * equals that forward's levels >= 1 bit for bit.  The workspace is mipnerf_b200_workspace_bytes', the precisions and
 * num_samples the forward's.  num_levels < 2: MIPNERF_B200_EINVAL.  The refusals, in order: the config, num_levels, the
 * weights, the rays, outs, t_prev / w_prev, then the forward's. */
int mipnerf_b200_forward_proposed(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                                  const mipnerf_b200_rays* rays, const float* t_prev, const float* w_prev,
                                  int randomized, const float* u_jitter, int white_bkgd, int precision,
                                  mipnerf_b200_level_out* outs, void* workspace, size_t workspace_bytes,
                                  void* stream);
int mipnerf_b200_forward_proposed_rng(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                                      const mipnerf_b200_rays* rays, const float* t_prev, const float* w_prev,
                                      const mipnerf_b200_rng* rng, int white_bkgd, int precision,
                                      mipnerf_b200_level_out* outs, void* workspace, size_t workspace_bytes,
                                      void* stream);

/* The uniforms those kernels draw: out[num_rays, ncols] for `stream_id` (0: t_rand in [0,1); >= 1: u_jitter in
 * [0, 1/ncols - eps)).  forward(t_rand = stream 0, u_jitter = stream 1+level) reproduces forward_rng bit for bit. */
int mipnerf_b200_philox_uniform(const mipnerf_b200_rng* rng, int stream_id, int64_t num_rays, int ncols, float* out,
                                void* stream);
/* The standard normals the _rng entry points add (times cfg->density_noise) to the raw density of level `level`
 * (models/mip_nerf.py:232-233): out[num_rays, num_samples].  Passed as outs[level].density_normal to the injected-
 * noise entry points they reproduce the in-kernel draws bit for bit. */
int mipnerf_b200_philox_normal(const mipnerf_b200_rng* rng, int level, int64_t num_rays, int num_samples, float* out,
                               void* stream);

/* distloss (models/mip.py:8-20), forward value per ray: weights [B,N], samples [B,N+1] (sorted) ->
 * per_ray_loss [B] = (1/3) sum_i d_i w_i^2 + sum_ij w_i w_j |m_i - m_j|; the reference's scalar is its mean. */
int mipnerf_b200_distloss(const float* weights, const float* samples, int64_t num_rays, int num_samples,
                          float* per_ray_loss, void* stream);

/* ---- training step (SURVEY.md §8f N2) -------------------------------------------------------------
 * Gradient buffers, one per entry of mipnerf_b200_weights.linears (same order and shapes). */
typedef struct mipnerf_b200_linear_grad {
  float* weight_grad; /* [out_features, in_features] */
  float* bias_grad;   /* [out_features]              */
} mipnerf_b200_linear_grad;

/* The loss of MipNeRFSystem.training_step (models/nerf_system.py:95-121):
 *   loss = sum_l  level_mse_mult[l] * sum_r mask_r |comp_rgb_l,r - target_r|^2 / mask_sum
 *               + level_dist_mult[l] * dist_scale * sum_r distloss_l,r
 * (reference: mse_mult = {coarse_loss_mult, 1}, dist_mult = {0.01*coarse_loss_mult, 0.01},
 * mask = rays.lossmult or ones, dist_scale = 1/B: the .mean() of models/mip.py:16,19).
 * `mask_sum` and `dist_scale` are over the GLOBAL batch so that ray shards of one batch (chunks, ranks)
 * produce gradients that simply add up. */
typedef struct mipnerf_b200_loss {
  const float* target_rgb;      /* [B,3] device                                                      */
  const float* lossmult;        /* [B] device, or NULL for a mask of ones                            */
  const float* mask_sum;        /* device scalar                                                     */
  float dist_scale;
  const float* level_mse_mult;  /* HOST [num_levels]                                                 */
  const float* level_dist_mult; /* HOST [num_levels]                                                 */
  float* per_ray_sqerr;         /* [num_levels, B] device, nullable: mask_r |comp_rgb - target|^2    */
  float* per_ray_distloss;      /* [num_levels, B] device, nullable                                  */
} mipnerf_b200_loss;

/* Workspace of the training step for every non-split precision (FP32, BF16, FP16): the largest of
 * mipnerf_b200_train_workspace_bytes_for over the three.  0 for configs the training step does not take. */
size_t mipnerf_b200_train_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_rays);
/* Workspace of the training step in one precision.  BF16X3 (chunks of 2048 rays, 5.7 GiB at the default
 * architecture, the 16-bit step's 4096-ray chunk 6.3 GiB) is non-zero only for the configs its fused step takes. */
size_t mipnerf_b200_train_workspace_bytes_for(const mipnerf_b200_config* cfg, int64_t num_rays, int precision);

/* MipNerf.forward (outputs in `outs`, as mipnerf_b200_forward) followed by the backward pass of the loss
 * above into `grads` (overwritten, or added to when `accumulate` != 0).  Replaces
 * `loss = training_step(...); loss.backward()` (models/nerf_system.py:95-121 + autograd).  Fenceposts carry
 * no gradient (stop_resample_grad=True semantics, models/mip.py:250-264).  precision FP32: every GEMM in fp32 FFMA
 * (the parity mode); BF16 / FP16: forward, dgrad and wgrad GEMMs of the 128- and 256-wide layers on wgmma with
 * 16-bit operands, heads / rendering in fp32.  The fused step (level kernels + 16-bit activation tile images) runs for
 * the level kernel's shapes (the default architecture and encodings, 128 samples only) with at most two levels; other
 * shapes with the default widths and encoding sizes (96-d IPE, 27-d view encoding) and net_depth <= 16 run per-layer
 * GEMMs on fp32 activations.  BF16X3 (the fused step only, at the same shapes; workspace from
 * mipnerf_b200_train_workspace_bytes_for): every operand of the forward, dgrad and wgrad GEMMs is split into bf16 hi +
 * lo halves (16 significant bits, fp32's range) and each product is hi.hi + lo.hi + hi.lo into fp32; gradients land an
 * order of magnitude closer to FP32's than BF16's.  FP16X3 is forward-only: MIPNERF_B200_EUNSUPPORTED, as is BF16X3 at
 * other shapes. */
int mipnerf_b200_forward_backward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* weights,
                                  const mipnerf_b200_rays* rays, int randomized, const float* t_rand,
                                  const float* u_jitter, int white_bkgd, int precision,
                                  const mipnerf_b200_loss* loss, mipnerf_b200_level_out* outs,
                                  const mipnerf_b200_linear_grad* grads, int num_grads, int accumulate,
                                  void* workspace, size_t workspace_bytes, void* stream);
/* randomized=True training step with the in-kernel generator (what a training loop calls every step). */
int mipnerf_b200_forward_backward_rng(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* weights,
                                      const mipnerf_b200_rays* rays, const mipnerf_b200_rng* rng, int white_bkgd,
                                      int precision, const mipnerf_b200_loss* loss, mipnerf_b200_level_out* outs,
                                      const mipnerf_b200_linear_grad* grads, int num_grads, int accumulate,
                                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- backward pass of MipNerf.forward for any loss (autograd) ----------------------------------------
 * Cotangents d L / d output of one level's rendered outputs; any pointer may be NULL (= zero). */
typedef struct mipnerf_b200_level_cotangent {
  const float* d_comp_rgb; /* [B,3] */
  const float* d_distance; /* [B]   */
  const float* d_acc;      /* [B]   */
  const float* d_weights;  /* [B,N] */
} mipnerf_b200_level_cotangent;

/* Gradients of  L = sum_l <cots[l], (comp_rgb, distance, acc, weights)_l>  with respect to the MLP tensors, into
 * `grads` (overwritten, or added to when `accumulate` != 0; same layout as mipnerf_b200_forward_backward).  The MLP
 * is re-evaluated at the fenceposts a forward produced, `t_samples[l]` [B,N+1] (read only; they carry no gradient,
 * stop_resample_grad=True), with the density noise of that forward: in-kernel Philox when `rng` is given (the
 * forward's seed / offset), else density_normal[l] [B,N] (required when randomized and cfg->density_noise > 0).
 * `randomized` only selects the density noise.  Same 4096-ray chunking and workspace as the training step
 * (mipnerf_b200_train_workspace_bytes).  precision FP32 or BF16; FP16 is refused (its fixed gradient scale is sized
 * for the training loss), the split precisions are refused (BF16X3 trains through mipnerf_b200_forward_backward only). */
int mipnerf_b200_backward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* weights,
                          const mipnerf_b200_rays* rays, const float* const* t_samples, int randomized,
                          const mipnerf_b200_rng* rng, const float* const* density_normal, int white_bkgd,
                          int precision, const mipnerf_b200_level_cotangent* cots,
                          const mipnerf_b200_linear_grad* grads, int num_grads, int accumulate, void* workspace,
                          size_t workspace_bytes, void* stream);

/* Gradient of distloss with respect to the weights (samples are constants):
 * d_weights[r,i] = grad_out[0] * scale * d per_ray_loss_r / d w_ri  (grad_out: device scalar, NULL = 1; the
 * reference's .mean() is scale = 1/num_rays). */
int mipnerf_b200_distloss_backward(const float* weights, const float* samples, int64_t num_rays, int num_samples,
                                   const float* grad_out, float scale, float* d_weights, void* stream);

/* mip-NeRF 360's interlevel loss, which trains proposal weights to cover the fine weights.  Per ray: fine fenceposts
 * t [B, n+1] and weights w [B, n], proposal fenceposts t_hat [B, n_hat+1] and weights w_hat [B, n_hat], n, n_hat >= 1
 * (neither needs to be sorted).  With C_0 = 0, C_{k+1} = C_k + w_hat_k (M = n_hat), for fine interval i:
 *   lo_i = clamp(#{k : t_hat_k <= t_i} - 1, 0, M),  hi_i = clamp(#{k : t_hat_k < t_{i+1}}, 0, M)  (exact fp32
 *   comparisons; for sorted fenceposts, the proposal intervals that overlap fine interval i),
 *   bound_i = C_{hi_i} - C_{lo_i} (0 when hi_i <= lo_i),
 *   per_ray_loss[r] = sum_i max(0, w_i - bound_i)^2 / (w_i + FLT_EPSILON),
 * in fp64, rounded once to fp32.  The result is bit for bit the same across runs and across any split of the rays into
 * calls.  The refusals, in order: num_rays < 0, a NULL tensor when num_rays > 0, then n or n_hat < 1. */
int mipnerf_b200_interlevel_loss(const float* t, const float* w, int n, const float* t_hat, const float* w_hat,
                                 int n_hat, int64_t num_rays, float* per_ray_loss, void* stream);
/* Its gradient with respect to w_hat (t, w and t_hat are constants: the paper's stop-gradient), written:
 *   d_w_hat[r, j] = grad_out[0] * scale * sum_{i : lo_i <= j < hi_i} -2 max(0, w_i - bound_i) / (w_i + FLT_EPSILON)
 * (grad_out: device scalar, NULL = 1; the mean over rays is scale = 1/num_rays), the sum in fp64 in increasing i.  The
 * same determinism and refusals as the loss, with d_w_hat in place of per_ray_loss.  No synchronisation. */
int mipnerf_b200_interlevel_loss_backward(const float* t, const float* w, int n, const float* t_hat,
                                          const float* w_hat, int n_hat, int64_t num_rays, const float* grad_out,
                                          float scale, float* d_w_hat, void* stream);

/* Stand-alone tensor-core linear layer  y[m,n] = act(x[m,k] . weight[n,k]^T + bias)  (wgmma, 16-bit operands, fp32
 * accumulate; n in {128,256}, k in {96,128,256}): the GEMM the training step uses for its forward and dgrad passes in
 * BF16 / FP16 mode.  `scratch` receives the packed weight image (n * ceil(k/64) * 128 bytes). */
int mipnerf_b200_linear_tc(const float* x, const float* weight, const float* bias, float* y, int64_t m, int n,
                           int k, int relu, int precision, void* scratch, size_t scratch_bytes, void* stream);

/* Stand-alone tensor-core weight gradient of one nn.Linear (what loss.backward() accumulates into layer.weight.grad /
 * layer.bias.grad, models/nerf_system.py:108-111):  dw[n, k1+k2] = dy[m,n]^T . [x1[m,k1] | x2[m / x2_row_div, k2]],
 * db[n] = column sums of dy; n in {128,256}, 16-bit operands rounded while staging, fp32 accumulation, per-slice
 * partials reduced in a fixed order (bit-reproducible).  x2 may be NULL (k2 = 0).  With k2 > 0, k1 must be a multiple
 * of 256 (MIPNERF_B200_EUNSUPPORTED otherwise); dy must be 16-byte aligned (MIPNERF_B200_EINVAL otherwise). */
size_t mipnerf_b200_wgrad_tc_scratch_bytes(int n, int k);
int mipnerf_b200_wgrad_tc(const float* dy, int n, const float* x1, int k1, const float* x2, int k2, int x2_row_div,
                          int64_t m, float* dw, float* db, int precision, void* scratch, size_t scratch_bytes,
                          void* stream);

/* The bf16x3 training step's GEMMs on their own, for tests: the fp32 operands are split into bf16 hi + lo tile images
 * and run through the step's kernels.  linear_x3: y[m,n] = [mask > 0] * (x[m,k] . weight[n,k]^T + r1[m] r1w[n]) (mask,
 * r1 nullable; r1 needs m % 128 == 0), y = hi + lo of the output images; n, k in {128, 256}.  wgrad_x3: as
 * mipnerf_b200_wgrad_tc; x2 is split into images when x2_row_div == 1 and read as fp32 rows otherwise (then
 * x2_row_div % 64 == 0 and m % 128 == 0). */
size_t mipnerf_b200_linear_x3_scratch_bytes(int64_t m, int n, int k);
int mipnerf_b200_linear_x3(const float* x, const float* weight, const float* r1, const float* r1w, const float* mask,
                           float* y, int64_t m, int n, int k, void* scratch, size_t scratch_bytes, void* stream);
size_t mipnerf_b200_wgrad_x3_scratch_bytes(int64_t m, int n, int k1, int k2, int x2_row_div);
int mipnerf_b200_wgrad_x3(const float* dy, int n, const float* x1, int k1, const float* x2, int k2, int x2_row_div,
                          int64_t m, float* dw, float* db, void* scratch, size_t scratch_bytes, void* stream);

/* torch.optim.Adam.step() for one flat fp32 tensor (models/nerf_system.py:70-72; amsgrad off, no weight
 * decay): `step` is the 1-based step count after this update; the gradient is read as grad * grad_scale
 * (1/world_size after a sum all-reduce). */
int mipnerf_b200_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                           double lr, double beta1, double beta2, double eps, int64_t step, double grad_scale,
                           void* stream);
/* The same update for `count` tensors that share lr / betas / eps / step (one optimiser group) in ONE launch; the
 * arrays are host arrays of device pointers / element counts. */
int mipnerf_b200_adam_step_multi(int count, float* const* params, const float* const* grads, float* const* exp_avg,
                                 float* const* exp_avg_sq, const int64_t* sizes, double lr, double beta1, double beta2,
                                 double eps, int64_t step, double grad_scale, void* stream);

/* Pinhole rays of rows [row0,row0+rows) of an H x W frame generated on the device, replacing the
 * host NumPy loaders (datasets/datasets.py:214-263, render_video.py:29-105).  `c2w_host` is a HOST
 * pointer to the row-major [3,4] camera-to-world matrix; outputs are [rows*W, 3|1] device buffers. */
int mipnerf_b200_generate_rays(const float* c2w_host, int height, int width, float focal, float near,
                               float far, int row0, int rows, float* origins, float* directions,
                               float* viewdirs, float* radii, float* near_out, float* far_out,
                               void* stream);

/* eval_errors (utils/metrics.py:190-197) of one rendered frame: pred / target [H, W, C] fp32 row-major (the layout
 * render_image produces) -> out[0] = PSNR = -10 log10(mean squared error) (utils/metrics.py:182-188), out[1] = mean
 * SSIM with the reference's 11x11 Gaussian window (sigma 1.5, zero padding, C1 = 0.01^2, C2 = 0.03^2; :44-126),
 * out[2] = the mean squared error.  `scratch`: mipnerf_b200_image_metrics_scratch_bytes() bytes. */
size_t mipnerf_b200_image_metrics_scratch_bytes(int height, int width, int channels);
int mipnerf_b200_image_metrics(const float* pred, const float* target, int height, int width, int channels,
                               void* scratch, size_t scratch_bytes, float* out, void* stream);

/* Training rays from pixel ids, scene resident in HBM (replaces the per-pixel host arrays of
 * datasets/datasets.py:116-168, 216-263 and the DataLoader's H2D copies, SURVEY.md §8f N4):
 *   cam_table [num_images, 24] = pix2cam (3x3 row-major, maps (x+.5, y+.5, 1) to a camera direction) |
 *                                cam2world (3x4 row-major) | lossmult | near | far
 *   offsets [num_images+1] first atlas row of each image; widths [num_images]; atlas [P,3] target colours
 *   pixel_ids [count] atlas rows (ids outside [0, offsets[num_images]) are clamped to the first / last row)
 *   -> the seven Rays fields ([count,3|1]) and rgb [count,3] (nullable). */
int mipnerf_b200_rays_from_pixels(const float* cam_table, const int64_t* offsets, const int32_t* widths,
                                  int num_images, const int64_t* pixel_ids, int64_t count, const float* atlas,
                                  float* origins, float* directions, float* viewdirs, float* radii,
                                  float* lossmult, float* near_out, float* far_out, float* rgb, void* stream);

/* ---- per-stage entry points (unit parity against the functions of models/mip.py) ---- */

/* sample_along_rays (models/mip.py:127-165): t_samples [B,N+1], means/covs [B,N,3] (nullable). */
int mipnerf_b200_sample_along_rays(const mipnerf_b200_rays* rays, int num_samples, int randomized,
                                   int disparity, const float* t_rand, float* t_samples,
                                   float* means, float* covs, void* stream);

/* cast_rays, cone + diagonal (models/mip.py:81-103): t_samples [B,N+1] -> means, covs [B,N,3]. */
int mipnerf_b200_cast_rays(const mipnerf_b200_rays* rays, const float* t_samples, int num_samples,
                           float* means, float* covs, void* stream);

/* integrated_pos_enc, diagonal (models/mip.py:322-350): means, covs [M,3] -> out [M, 6*(max-min)].
 * -60 <= min_deg <= max_deg <= 60 (here and in pos_enc); an empty range is an [M, 0] output. */
int mipnerf_b200_integrated_pos_enc(const float* means, const float* covs, int64_t num_points,
                                    int min_deg, int max_deg, float* out, void* stream);

/* pos_enc (models/mip.py:353-363): x [B,3] -> out [B, 6*(max-min) (+3)]. */
int mipnerf_b200_pos_enc(const float* x, int64_t num_points, int min_deg, int max_deg,
                         int append_identity, float* out, void* stream);

/* MLP.forward (models/mip_nerf.py:75-111): x [B*N, xyz_dim], view_enc [B, view_dim] or NULL ->
 * raw_rgb [B*N,3], raw_density [B*N,1]. */
int mipnerf_b200_mlp_forward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                             const float* x, const float* view_enc, int64_t num_rays,
                             int samples_per_ray, int precision, float* raw_rgb, float* raw_density,
                             void* workspace, size_t workspace_bytes, void* stream);

size_t mipnerf_b200_mlp_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_rays,
                                        int samples_per_ray, int precision);

/* volumetric_rendering (models/mip.py:366-401): rgb [B,N,3], density [B,N,1] already activated.
 * num_samples N in {32, 64, 96, 128, 192, 256} (the forward's set); any other N >= 1 is EUNSUPPORTED. */
int mipnerf_b200_volumetric_rendering(const float* rgb, const float* density,
                                      const float* t_samples, const float* dirs, int64_t num_rays,
                                      int num_samples, int white_bkgd, float* comp_rgb,
                                      float* distance, float* acc, float* weights, void* stream);

/* sorted_piecewise_constant_pdf (models/mip.py:168-229): bins [B,nb+1], weights [B,nb] (NOT
 * modified) -> samples [B,num_samples]; inds (nullable) are the searchsorted(right=True) results.
 * num_bins nb a multiple of 32, <= 512 (EUNSUPPORTED otherwise: above 544 bins CPU torch sums a row in another
 * order, so the samples would stop being bit-exact); num_samples >= 2. */
int mipnerf_b200_sorted_piecewise_constant_pdf(const float* bins, const float* weights,
                                               int64_t num_rays, int num_bins, int num_samples,
                                               int randomized, const float* u_jitter,
                                               float* samples, int64_t* inds, void* stream);

/* resample_along_rays (models/mip.py:232-280): blur-pool + padding + inverse CDF + cast_rays.
 * t_samples [B,N+1], weights [B,N] -> new_t_samples [B,N+1], means/covs [B,N,3] (nullable), inds [B,N+1] (nullable);
 * num_samples N a multiple of 32, <= 512 (EUNSUPPORTED otherwise, as for sorted_piecewise_constant_pdf). */
int mipnerf_b200_resample_along_rays(const mipnerf_b200_rays* rays, const float* t_samples,
                                     const float* weights, int num_samples, int randomized,
                                     const float* u_jitter, float resample_padding,
                                     float* new_t_samples, float* means, float* covs, int64_t* inds,
                                     void* stream);

/* ---- density queries and meshes ----
 * Density of the field at Gaussians: means [P,3], diagonal covs [P,3] (NULL: zero covariance, i.e. plain positional
 * encoding) -> the IPE (models/mip.py:322-350) -> trunk (layers 0-7, skip after 4) -> density_layer
 * (models/mip_nerf.py:93-98).  raw_density [P] = MLP.forward's raw density (no noise); density [P] =
 * softplus(raw + cfg->density_bias).  Either output may be NULL, not both; cfg->disable_integration zeroes covs.
 * FP32 takes any config check_config accepts; the tensor-core precisions the configs the forward takes on the tensor
 * cores (see the precision list above), through the density-only mode of the level kernel.  Points run in launch
 * chunks; results do not depend on how a query is split. */
size_t mipnerf_b200_density_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_points, int precision);
int mipnerf_b200_query_density(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                               const float* covs, int64_t num_points, int precision, float* raw_density,
                               float* density, void* workspace, size_t workspace_bytes, void* stream);

/* Radiance of the field at Gaussians, each seen from its own direction: means / covs as for the density query,
 * viewdirs [P,3] (encoded as given; the reference encodes unit directions) -> MLP.forward(x [P,1,xyz_dim],
 * pos_enc(viewdirs) [P,view_dim]) (models/mip_nerf.py:75-111).  raw_rgb [P,3] / raw_density [P] are its raw heads (no
 * noise); rgb [P,3] = sigmoid(raw) * (1 + 2 rgb_padding) - rgb_padding and density [P] = softplus(raw +
 * cfg->density_bias).  Any output may be NULL, not all.  viewdirs may be NULL only when !cfg->use_viewdirs (FP32 only:
 * the colour head then reads the trunk output, as the reference's).  Refusals and precisions as for the density query.
 * The tensor-core precisions run the radiance mode of the level kernel; their workspace is two [128][128] fp32 slots
 * of view-direction terms per CTA of a launch, min(ceil(P / 128), 4096, SMs) CTAs, so it is sized by the device the
 * call runs on.  Results do not depend on how a query is split. */
size_t mipnerf_b200_radiance_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_points, int precision);
int mipnerf_b200_query_radiance(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                                const float* covs, const float* viewdirs, int64_t num_points, int precision,
                                float* raw_rgb, float* raw_density, float* rgb, float* density, void* workspace,
                                size_t workspace_bytes, void* stream);

/* Radiance of the field at Gaussians under one shared set of directions: means / covs [P,3] as for the density query,
 * dirs [D,3] (encoded as given), each point seen from every direction.  The view layer's pre-activation is split into
 * W_view[:, :256] . bottleneck(p) (per point) and b_view + W_view[:, 256:] . pos_enc(dir d) (per direction); per pair
 * remain the ReLU and the colour head.  Outputs, each may be NULL but not all:
 *   raw_rgb / rgb [P,D,3]: query_radiance's raw head / activation of (point p, direction d);
 *   raw_density / density [P]: query_density's;
 *   proj_out [P,num_basis,3] = sum over d = 0..D-1, in order, in fp32, of table[d][k] c[p][d] with c = raw_rgb when
 *   proj_raw, else rgb; table [D,num_basis] (device), num_basis 1..16.  Bit-reproducible, independent of chunking.
 * The tensor-core precisions take the configs query_radiance takes on the tensor cores and return query_radiance's
 * raw_rgb / rgb bit for bit (the view-accumulator mode of the level kernel, then the per-pair kernel in the level
 * kernel's summation order); FP32 takes use_viewdirs configs with one 128-wide view layer, within fp32 round-off of
 * query_radiance (the view layer's sum runs in another order).  use_viewdirs=0, num_dirs < 1, proj_out without table
 * or with num_basis outside 1..16: refused.  Workspace: one chunk of at most 524288 points (256 MB of view
 * accumulators on the tensor cores) plus D x 512 bytes. */
size_t mipnerf_b200_radiance_dirs_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_points, int64_t num_dirs,
                                                  int precision);
int mipnerf_b200_query_radiance_dirs(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                                     const float* covs, int64_t num_points, const float* dirs, int64_t num_dirs,
                                     int precision, float* raw_rgb, float* rgb, float* raw_density, float* density,
                                     const float* table, int num_basis, int proj_raw, float* proj_out,
                                     void* workspace, size_t workspace_bytes, void* stream);

/* ---- gradients of field queries with respect to the MLP tensors ----
 * Cotangents of one query's outputs; any pointer may be NULL (= zero). */
typedef struct mipnerf_b200_query_cotangent {
  const float* d_raw_rgb;      /* [P,3] */
  const float* d_raw_density;  /* [P]   */
  const float* d_rgb;          /* [P,3]  rgb = sigmoid(raw) (1 + 2 rgb_padding) - rgb_padding          */
  const float* d_density;      /* [P]    density = softplus(raw + density_bias), torch's threshold 20  */
} mipnerf_b200_query_cotangent;

/* Workspace of mipnerf_b200_query_backward for a radiance (radiance != 0) or density query of num_points points: one
 * chunk of at most 524288 points, so the size stops growing there.  0 where the backward refuses the config or
 * precision. */
size_t mipnerf_b200_query_backward_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_points,
                                                   int radiance, int precision);
/* Gradients of L = <cot, outputs of query_radiance (viewdirs != NULL) or query_density (viewdirs == NULL)> w.r.t. the
 * MLP tensors, into `grads` (same layout and accumulate semantics as mipnerf_b200_backward).  covs NULL or
 * cfg->disable_integration: zero covariance; no density noise.  The means, covs and viewdirs carry no gradient.  A
 * density query reads only d_raw_density and d_density, and writes exact zeros to the bottleneck, view-layer and
 * colour-head gradients (leaves them untouched when `accumulate` is set).
 * BF16 runs the query again on the level kernel's query mode with the training dump (the outputs and 16-bit activation
 * tiles are the forward query's own, bit for bit), then the fused training step's tile-image backward chain; it takes
 * the default architecture and encodings.  FP32 re-evaluates the query with its fp32 activations kept (the IPE stage
 * kernel, pos_enc, the fp32 MLP, the same values as the fp32 query) and runs the per-layer fp32 chain; it takes the
 * configs mipnerf_b200_backward takes.  FP16 (its fixed gradient scale is sized for the training loss), the split
 * precisions (forward-only here) and other configs: MIPNERF_B200_EUNSUPPORTED.  Points run in chunks of 524288 and the
 * wgrad partials are reduced in a fixed order: the gradients are bit-reproducible, though a query split into two calls
 * sums in a different order. */
int mipnerf_b200_query_backward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                                const float* means, const float* covs, const float* viewdirs, int64_t num_points,
                                int precision, const mipnerf_b200_query_cotangent* cot,
                                const mipnerf_b200_linear_grad* grads, int num_grads, int accumulate,
                                void* workspace, size_t workspace_bytes, void* stream);

/* Isosurface of a scalar grid [nz, ny, nx] fp32 (x fastest, every dimension >= 2) by marching tetrahedra (6 Kuhn
 * tetrahedra per cell): a watertight indexed mesh whose normals point from inside (value > iso; NaN is outside) to
 * outside.  Pass 1 writes counts[2] (device int64: vertices, faces); pass 2, with the same scratch, writes verts [V,3]
 * fp32 and faces [F,3] int32 (lo_host / hi_host: HOST float[3], the positions of lattice points 0 and n-1 per axis).
 * Vertex ids follow (lattice point in x-fastest order, edge direction x, y, z, x+y, x+z, y+z, x+y+z), faces (cell,
 * tetrahedron, triangle): the output is bit-reproducible.  Emit reads the vertex count back (one stream synchronise)
 * and answers MIPNERF_B200_EUNSUPPORTED when int32 indices cannot address it. */
size_t mipnerf_b200_isosurface_scratch_bytes(int nx, int ny, int nz);
int mipnerf_b200_isosurface_count(const float* grid, int nx, int ny, int nz, float iso, void* scratch,
                                  size_t scratch_bytes, int64_t* counts, void* stream);
int mipnerf_b200_isosurface_emit(const float* grid, int nx, int ny, int nz, const float* lo_host,
                                 const float* hi_host, float iso, const void* scratch, float* verts,
                                 int32_t* faces, void* stream);
/* Vertex normals of the mesh _emit wrote, from the same grid, bounds, iso and scratch (after _emit): normals [V,3] fp32,
 * vertex v's at row v.  The grid gradient at both ends of the vertex's lattice edge (central differences over 2 step
 * per axis, one-sided over step at the box faces), interpolated with the vertex's t, negated and normalised: the unit
 * direction from inside to outside, the faces' orientation.  (0, 0, 0) where that gradient is zero or not finite (a NaN
 * neighbour).  Every operation is explicitly rounded: the normals are bit-reproducible. */
int mipnerf_b200_isosurface_normals(const float* grid, int nx, int ny, int nz, const float* lo_host,
                                    const float* hi_host, float iso, const void* scratch, float* normals, void* stream);

/* ---- baked grids (mipnerf_pl_b200/baked.py): density and raw SH colour on nested lattices, rendered by ray marching */
#define MIPNERF_B200_GRID_MAX_LEVELS 4

/* One level of a baked grid: a lattice of nx * ny * nz points spanning the grid's bounds (point (i, j, k) at
 * lo + (i, j, k) * (hi - lo) / (n - 1)), x fastest. */
typedef struct mipnerf_b200_grid_level {
  const int32_t* cells; /* [nz, ny, nx, 2] per point: fp32 density (bit pattern), then the row of its SH coefficients
                           in `sh` (-1: not kept, coefficients 0) */
  const float* sh;      /* [M, (degree + 1)^2, 3] fp32 raw-colour SH coefficients of the kept points */
  int32_t nx, ny, nz;
} mipnerf_b200_grid_level;

/* Levels nest: level l has (n_0 - 1) / 2^l + 1 points per axis.  `occupancy` [oz, oy, ox] uint8 (o = ceil((n_0 - 1) /
 * block) per axis) marks the macro cells of block^3 finest cells where some level may interpolate to non-zero density;
 * a 0 cell is skipped.  lo / hi: the bounds; rgb_padding: colour = sigmoid(raw) (1 + 2 rgb_padding) - rgb_padding. */
typedef struct mipnerf_b200_grid {
  mipnerf_b200_grid_level levels[MIPNERF_B200_GRID_MAX_LEVELS];
  int32_t num_levels; /* 1..4 */
  int32_t degree;     /* 0..3, the field.sh_basis convention */
  float lo[3], hi[3];
  float rgb_padding;
  const uint8_t* occupancy;
  int32_t block; /* macro cell edge in finest cells, a multiple of 2^(num_levels - 1) */
} mipnerf_b200_grid;

/* Render rays through a baked grid (rays->viewdirs required): K = max(1, ceil((far - near) |d| / step)) intervals of
 * dt = (far - near) / K, samples at t_k = near + (k + 1/2) dt (K, dt, t_k in fp32), delta = dt |d|.  A sample at
 * x = o + t_k d (fp32) outside [lo, hi] has density 0; inside, level lambda = clamp(log2(sqrt(3) radii t_k / s_0), 0,
 * L - 1) (s_0: the finest level's largest voxel edge) blends the trilinear density and SH coefficients of levels
 * floor(lambda) and floor(lambda) + 1.  Compositing as mipnerf_b200_volumetric_rendering (distance not divided by acc,
 * clamped to [near, far]), stopping after the first sample that leaves the transmittance below 1e-4.  Empty macro cells
 * are skipped without moving the samples, so the result equals marching every sample bit for bit.  rgb [B,3], distance
 * [B], acc [B].  No allocation, no synchronisation. */
int mipnerf_b200_grid_render(const mipnerf_b200_grid* grid, const mipnerf_b200_rays* rays, float step, int white_bkgd,
                             float* rgb, float* distance, float* acc, void* stream);

/* The SH rows of a baked grid quantized to 8 bits (mipnerf_pl_b200/baked.py, BakedGrid.quantize): per level and per
 * (coefficient k, channel), an affine code with offset = the column's minimum and scale = (max - min) / 255, so
 * rows[l][r, k, ch] = clamp(round((c - offset) / scale), 0, 255) (0 for a constant column, scale 0).  Coefficient k,
 * channel ch of a row reads as deq(q) = fl32(fl32(float(q) * scale[l][k][ch]) + offset[l][k][ch]): two explicitly
 * rounded fp32 operations, no fused multiply-add.  scale and offset are values in the struct, not device pointers;
 * entries past (degree + 1)^2 and num_levels are not read. */
typedef struct mipnerf_b200_grid_sh_u8 {
  const uint8_t* rows[MIPNERF_B200_GRID_MAX_LEVELS]; /* [M_l, (degree + 1)^2, 3] uint8; NULL: no kept points */
  float scale[MIPNERF_B200_GRID_MAX_LEVELS][16][3];  /* [level][k][channel], k < (degree + 1)^2 */
  float offset[MIPNERF_B200_GRID_MAX_LEVELS][16][3];
} mipnerf_b200_grid_sh_u8;

/* mipnerf_b200_grid_render on a grid whose SH rows are `sh`'s uint8 rows: the same march, skipping, level blend and
 * compositing, with every SH coefficient read as deq(q) above, in the same order and accumulation as the fp32 rows.
 * So rgb, distance and acc equal, bit for bit, mipnerf_b200_grid_render's on the grid whose levels[l].sh are the
 * dequantized rows; distance and acc equal the unquantized grid's, since the density path does not read the rows.
 * Every levels[l].sh must be NULL (the rows read are sh->rows[l]), and scale / offset must be finite for every level and
 * coefficient in use.  The scale / offset tables are passed to the kernel by value: no allocation, no copy, no
 * synchronisation. */
int mipnerf_b200_grid_render_u8(const mipnerf_b200_grid* grid, const mipnerf_b200_grid_sh_u8* sh,
                                const mipnerf_b200_rays* rays, float step, int white_bkgd, float* rgb, float* distance,
                                float* acc, void* stream);

/* The cells of a baked grid stored as bricks of 8 x 8 x 8 lattice points (mipnerf_pl_b200/baked.py,
 * BakedGrid.sparsify), in place of levels[l].cells.  Level l's table is [tz, ty, tx] int32 with t = ceil(n / 8) per
 * axis of that level: brick (bi, bj, bk)'s id in the pool, or -1 for a brick not stored.  The pool is [num_bricks, 8,
 * 8, 8, 2] int32: brick b's point (z, y, x), x fastest, holds the word levels[l].cells holds, (density bits, SH row).
 * Lattice point (i, j, k) lives in brick (i >> 3, j >> 3, k >> 3) at (k & 7, j & 7, i & 7).  A brick not stored reads
 * (+0.0 bits, -1) at every point, so a grid whose bricks holding any other word are all stored renders exactly as
 * its dense cells.  The pool may be NULL for a level whose table holds only -1. */
typedef struct mipnerf_b200_grid_bricks {
  const int32_t* table[MIPNERF_B200_GRID_MAX_LEVELS];
  const int32_t* pool[MIPNERF_B200_GRID_MAX_LEVELS];
} mipnerf_b200_grid_bricks;

/* mipnerf_b200_grid_render (sh_u8 NULL: fp32 rows in levels[l].sh) or mipnerf_b200_grid_render_u8 (sh_u8 non-NULL,
 * every levels[l].sh NULL) on a grid whose cells are `bricks`: every levels[l].cells must be NULL and every
 * bricks->table[l] non-NULL.  The same march, skipping, level blend, row reads and compositing, so rgb, distance and
 * acc equal, bit for bit, the dense render of the cells the bricks encode.  No allocation, no synchronisation. */
int mipnerf_b200_grid_render_bricks(const mipnerf_b200_grid* grid, const mipnerf_b200_grid_bricks* bricks,
                                    const mipnerf_b200_grid_sh_u8* sh_u8, const mipnerf_b200_rays* rays, float step,
                                    int white_bkgd, float* rgb, float* distance, float* acc, void* stream);

/* Per-level gradient buffers of a baked grid's parameters: density[l] [M_l] is indexed by SH row (the density of the
 * kept point whose row is r), sh[l] [M_l, (degree + 1)^2, 3] has the layout of levels[l].sh.  Dropped points (row -1)
 * are not parameters. */
typedef struct mipnerf_b200_grid_grads {
  float* density[MIPNERF_B200_GRID_MAX_LEVELS];
  float* sh[MIPNERF_B200_GRID_MAX_LEVELS];
} mipnerf_b200_grid_grads;

/* The derivative of mipnerf_b200_grid_render's outputs (same grid, rays, step and white_bkgd) under the cotangents
 * d_rgb [B,3], d_distance [B], d_acc [B] (each may be NULL: zero) with respect to the kept points' densities and SH
 * coefficients, ADDED into `grads` (the caller zeroes it; density[l] and sh[l] are required for every level whose
 * levels[l].sh is non-NULL).  It differentiates the marcher as it runs: the same fp32 sample lattice, inside test,
 * level choice and blend, trilinear corner weights, the sigmoid with rgb_padding, white_bkgd, and the distance clamp
 * (the gradient passes where near <= distance <= far).  Samples outside the bounds, in empty macro cells, or after the
 * one that stops the ray contribute nothing.  A sample of an occupied cell whose density interpolates to exactly 0
 * does contribute to the density of its kept corners.  On a grid straight from the baker, every corner a sample in an
 * empty cell reads is a dropped point, so skipping empty cells loses no gradient up to rounding at cell faces; once
 * kept densities have been set to 0 (and the occupancy rebuilt from them) the skip can drop the gradient that would
 * let those densities grow back.  The scatter is fp32 atomic adds: reproducible to round-off, not bit for bit.  No
 * allocation, no synchronisation. */
int mipnerf_b200_grid_render_backward(const mipnerf_b200_grid* grid, const mipnerf_b200_rays* rays, float step,
                                      int white_bkgd, const float* d_rgb, const float* d_distance, const float* d_acc,
                                      const mipnerf_b200_grid_grads* grads, void* stream);

/* The visibility of a baked grid's kept points over a batch of rays, for pruning (PlenOctrees): per kept point the
 * largest score it receives from any composited sample.  The march is mipnerf_b200_grid_render's for density only
 * (same samples, skipping, level blend and trilinear weights, same stop after the sample that leaves the transmittance
 * below 1e-4).  At a composited sample of blending weight w_k = T_k alpha_k (formed as the renderer forms it), a kept
 * corner c of level l scores w_k * (lw * wc_c): wc_c is its trilinear weight and lw the level weight (1 - f for level
 * floor(lambda), 1 when f == 0, f for level floor(lambda) + 1), so lw * wc_c is the coefficient the renderer gives the
 * corner's colour.  max_weight holds num_levels pointers; entry l has M_l floats in SH-row order (required for every
 * level whose levels[l].sh is non-NULL).  The call RAISES each entry to the maximum of its current value and every
 * score from these rays: the caller initialises the entries to 0, and calls over batches of rays accumulate.  The
 * maximum is an integer atomicMax on the float bits (valid as scores are >= 0; a negative score from a negative
 * density never raises an entry from 0), so the result is bit-reproducible: across runs, across any split of the rays
 * into calls and under any permutation of the rays.  A prune holds for renders at the step it was computed with.  No
 * allocation, no synchronisation. */
int mipnerf_b200_grid_visibility(const mipnerf_b200_grid* grid, const mipnerf_b200_rays* rays, float step,
                                 float* const* max_weight, void* stream);

/* mipnerf_b200_grid_visibility on a grid whose cells are `bricks` (every levels[l].cells NULL, every bricks->table[l]
 * non-NULL, as for mipnerf_b200_grid_render_bricks): the same march and scores, so max_weight equals, bit for bit, the
 * dense call's on the cells the bricks encode.  The SH rows are not read, so levels[l].sh may be NULL on a grid whose
 * rows are not baked yet (the streamed bake prunes before it bakes them); max_weight[l] is required for every level
 * whose bricks->pool[l] is non-NULL.  No allocation, no synchronisation. */
int mipnerf_b200_grid_visibility_bricks(const mipnerf_b200_grid* grid, const mipnerf_b200_grid_bricks* bricks,
                                        const mipnerf_b200_rays* rays, float step, float* const* max_weight,
                                        void* stream);

/* Proposal weights from a baked grid's density (mip-NeRF 360's proposal sampling): the level-0 weights of a forward at
 * the caller's fenceposts t_samples [B, N+1], for mipnerf_b200_forward_proposed.  Per ray and interval i, in fp32:
 *   t_mid = fl(fl(t_i + t_{i+1}) * 0.5), x = fl(o + fl(t_mid d)) per axis, delta_i = fl(fl(t_{i+1} - t_i) |d|) with
 *   |d| = fl(sqrt(fl(fl(dx dx + dy dy) + dz dz))) (every operation rounded once, as the renderer's sample lattice);
 *   sigma_i = the renderer's density at x: 0 outside [lo, hi], else levels floor(lambda) and floor(lambda) + 1 blended
 *   by lambda = clamp(log2(sqrt(3) radii t_mid / s_0), 0, L - 1), each trilinear over its lattice (0 at dropped points);
 *   s_i = fl(sigma_i delta_i), w_i = fl(fl(1 - exp(-s_i)) exp(-S_i)), S_i = sum_{j<i} s_j accumulated in order in fp32:
 *   volumetric_rendering's weights (models/mip.py:366-401), every interval weighted (no early stop).
 * Midpoints in empty macro cells are not looked up (their density is exactly 0), so the weights equal those of the
 * grid with every macro cell occupied bit for bit.  bricks NULL: the cells are levels[l].cells; otherwise the cells
 * are `bricks` (as mipnerf_b200_grid_render_bricks: every levels[l].cells NULL, every bricks->table[l] set), with the
 * same weights bit for bit as the dense cells they encode.  No SH row and no viewdir is read.  The refusals, in order:
 * grid NULL, the rays, t_samples / weights NULL, num_samples outside 1..256, bricks' cells, then the grid.  No
 * allocation, no synchronisation. */
int mipnerf_b200_grid_proposal(const mipnerf_b200_grid* grid, const mipnerf_b200_grid_bricks* bricks,
                               const mipnerf_b200_rays* rays, const float* t_samples, int num_samples, float* weights,
                               void* stream);

/* The derivative of sum_{r,i} d_weights[r,i] w[r,i], w = mipnerf_b200_grid_proposal's weights (same grid, rays and
 * t_samples [B, num_samples+1]), with respect to the kept points' densities, ADDED into grads->density (the caller
 * zeroes it; required for every level whose levels[l].sh is non-NULL).  grads->sh is not read.  Dense fp32 cells only
 * (levels[l].cells): a trainable grid is dense.  Per ray, with g_i = d_weights[r,i], s_i = sigma_i delta_i and S_i =
 * sum_{j<i} s_j, so that w_i = e^{-S_i} - e^{-S_{i+1}}:
 *   dL/ds_k = g_k e^{-S_{k+1}} - sum_{i>k} g_i w_i,   dL/dsigma_k = delta_k dL/ds_k,
 * each w_i recomputed with the forward's fp32 expressions and the suffix formed as total - prefix, then scattered
 * through the level blend and trilinear weights into the kept corners.  A midpoint outside the bounds or in an empty
 * macro cell (which the forward does not look up) gets no gradient.  So the gradient can raise density only at kept
 * points whose midpoints fall in occupied macro cells: empty space stays empty.  The scatter is fp32 atomic adds:
 * reproducible to round-off, not bit for bit.  The refusals, in order: grid NULL, the rays, t_samples / d_weights /
 * grads NULL (when num_rays > 0), num_samples outside 1..256, the grid, then a NULL grads->density[l] (when
 * num_rays > 0).  No allocation, no synchronisation. */
int mipnerf_b200_grid_proposal_backward(const mipnerf_b200_grid* grid, const mipnerf_b200_rays* rays,
                                        const float* t_samples, int num_samples, const float* d_weights,
                                        const mipnerf_b200_grid_grads* grads, void* stream);

/* The total-variation prior of a baked grid (Plenoxels), for fine-tuning.  Per level l, on that level's own lattice:
 * for each kept point p (SH row r, lattice position points[l][r] = i + nx (j + ny k), r < num_points[l] = M_l) and
 * each axis a, q = p + e_a is its forward neighbour, and
 *   density:  D_a(p) = s(q) - sigma(p), s(q) = sigma(q) (the cell's density) when q is kept, 0 when it is dropped
 *             (the value the renderer interpolates there);
 *   SH:       D_a c_{k,ch}(p) = c_{k,ch}(q) - c_{k,ch}(p) when q is kept, 0 when q is dropped (it has no row);
 *   both are 0 where q lies outside the lattice.
 * Point p's terms are tv_density[l][r] = sqrt(eps + sum_a D_a(p)^2) and tv_sh[l][r] = sum_{k,ch} sqrt(eps + sum_a
 * (D_a c_{k,ch}(p))^2) (the k, ch sum in row order).  TV_density and TV_sh are their sums over every level's kept
 * points divided by M = sum_l M_l (0 when M = 0); that normalisation is the caller's.
 * With `grads`, the call WRITES (does not add) grads->density[l][r] = weights[0] * d(sum of density terms) /
 * dsigma(p) and grads->sh[l][r] = weights[1] * d(sum of SH terms) / dc(p), the sums over every kept point of the
 * level.  `weights` is a device array of 2 fp32 (read only with grads).  Each entry is a fixed-order sum formed by one
 * thread, so the gradient is bit-reproducible.  Every output may be NULL: tv_density, tv_sh and grads themselves, and
 * any of their per-level pointers; a level whose outputs are all NULL is not read.  eps > 0 and finite.  The density
 * is read from levels[l].cells, the coefficients from levels[l].sh (required, with points[l], where M_l > 0).
 * points and num_points are host arrays of num_levels entries, points[l] a device int64 [M_l] array.  Every row id
 * in the cells must be < M_l.  No allocation, no synchronisation. */
int mipnerf_b200_grid_tv(const mipnerf_b200_grid* grid, const int64_t* const* points, const int64_t* num_points,
                         float eps, float* const* tv_density, float* const* tv_sh, const float* weights,
                         const mipnerf_b200_grid_grads* grads, void* stream);

/* Hardware self-test of the wgmma building blocks (descriptor / swizzle / accumulator-fragment conventions):
 * d[128,n] = a[128,k] . b[n,k]^T, 16-bit operands (precision BF16|FP16), fp32 accumulate; n in {128, 256}.
 * variant bit 0: B through a pre-swizzled image + cp.async.bulk (needs `scratch`); bit 1: A in registers (the RS form
 * of wgmma, k a multiple of 32); bit 2: one K = 32 slab in the 64-byte-swizzle layout; bit 3: A as 32-byte-swizzle
 * K = 16 blocks. */
int mipnerf_b200_selftest_umma(const float* a, const float* b, float* d, int n, int k, int precision,
                               int variant, void* scratch, size_t scratch_bytes, void* stream);

/* ---- launch accounting (bench.py: `gpu_launches`, live launch duration of the dominant kernel) ----
 * Every kernel launch of the library is counted per kernel id; with timing enabled each launch is
 * also bracketed by CUDA events on its stream.  profile_read synchronises the pending events. */
int mipnerf_b200_profile_enable(int timing_on);
int mipnerf_b200_profile_num_kernels(void);
const char* mipnerf_b200_profile_kernel_name(int kernel_id);
int mipnerf_b200_profile_read(int kernel_id, int64_t* launches, double* timed_ms,
                              int64_t* timed_launches, int reset);

#ifdef __cplusplus
}
#endif
#endif /* MIPNERF_B200_H_ */
