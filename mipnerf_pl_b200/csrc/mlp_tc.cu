// mlp_tc.cu — the tensor-core path: one fused kernel per sampling level that does, per ray,
//   fenceposts (coarse, or resampled from the previous level)      (models/mip.py:127-165, 168-280)
//   -> conical-frustum Gaussians -> IPE features                   (models/mip.py:81-103, 322-350)
//   -> 8x256 trunk + density / bottleneck / view / colour heads    (models/mip_nerf.py:75-111)
//   -> activations + front-to-back alpha compositing               (models/mip_nerf.py:236-238, mip.py:366-401)
// without any intermediate tensor touching HBM.  Per level the kernel reads 52 B of ray data (+ the previous
// level's fenceposts / weights for the resampler) and writes t_samples/comp_rgb/distance/acc/weights; the weights
// stream from L2.  A forward is two launches of this kernel and nothing else.
// Kernel mapping: see mlp_level_kernel below.  Other mode of the same kernel: MLP-only (features from the caller, raw
// heads out: mipnerf_b200_mlp_forward).
#include "mlp_tc.h"

#include <algorithm>
#include <cstdlib>
#include <mutex>

#include "kernels.h"
#include "profile.h"
#include "ray_math.cuh"
#include "ray_resample.cuh"
#include "tc_common.cuh"

namespace mipnerf {
namespace {

using namespace tc;

constexpr int kN = 128;         // sample rows per tile (the M of a tile's GEMMs); a ray is kT = 1 or 2 tiles
constexpr int kWidth = 256;     // trunk width
constexpr int kCond = 128;      // view layer width
constexpr int kFeat = 96;       // IPE width
constexpr int kViewDim = 27;
constexpr int kNumLayers = 10;  // 8 trunk + extra_layer + view layer
constexpr uint32_t kStageBytes = 16384;  // A-operand slab: [128 x 64] 16-bit, SW128
constexpr uint32_t kTailBytes = 8192;    // feature tail slab: [128 x 32] 16-bit, SW64
constexpr uint32_t kABytes = 65536;      // 4 slabs
constexpr uint32_t kFBytes = kStageBytes + kTailBytes;  // feature tile: SW128 slab (K 0..63) + SW64 slab (K 64..95)
// Biases and the two CUDA-core heads, broadcast-read by every thread: constant bank.
struct SmallParams {
  float bias[9][kWidth];      // layers.0..7, extra_layer
  float w_density[kWidth];    // density_layer.weight
  float w_color[3][kCond];    // color_layer.weight
  float b_density;
  float b_color[3];
};
__constant__ SmallParams c_small;

// The weight stages.  The packed image holds, per layer and per N-half (rows h*128..), the layer's K extent as K-slabs
// in the order the producer streams them.  One K-slab is one weight stage: [128 rows x kw] 16-bit, K-major and
// pre-swizzled, so that loading it is one contiguous cp.async.bulk.
//   * bf16 / fp16 ("wide" stages): 64-wide K-slabs as [128 x 128 B] SW128 stages of 16 KB, four wgmma K steps per
//     commit group.  Layer 0 (K = 96) and layer 5 (K = 352 = [h | x]) end in a 32-wide [128 x 64 B] SW64 tail of 8 KB.
//   * split modes: 32-wide SW64 stages of 8 KB throughout; the hi and lo stages of a K-slab share one 16 KB ring slot.
//     Wide hi + lo stages would need 32 KB slots: the two-slot ring would add 32 KB to the split modes' 213 KB layout,
//     beyond the 227 KB a CTA may have.
// Per layer, the image has the same size in both.  The packer, the producer and the consumers take the layout from
// w_stage / w_stage_offset only.
__host__ __device__ constexpr int layer_k(int l) {  // the view layer's K is its 256 trunk columns (the view-direction
  return l == 0 ? kFeat : (l == 5 ? kWidth + kFeat : kWidth);  // columns go into the per-ray bias)
}
__host__ __device__ constexpr int num_halves(int l) { return l == 9 ? 1 : 2; }
__host__ __device__ constexpr int slab_width(bool wide) { return wide ? 64 : 32; }
__host__ __device__ constexpr int num_slabs(bool wide, int l) {
  return (layer_k(l) + slab_width(wide) - 1) / slab_width(wide);
}
struct WStage {
  int k0, kw;      // K offset and width: 64, or 32 (a wide layout's tail, or any split-mode stage)
  uint32_t bytes;  // 128 rows x kw 16-bit
  bool sw128;      // SW128 (kw = 64) or SW64 (kw = 32)
};
// K-slab s of either N-half of layer l
__host__ __device__ constexpr WStage w_stage(bool wide, int l, int s) {
  const int k0 = s * slab_width(wide), kw = wide && layer_k(l) - k0 < 64 ? 32 : slab_width(wide);
  return WStage{k0, kw, (uint32_t)kw * 256u, kw == 64};
}
static_assert(kFeat % 32 == 0 && kWidth % 64 == 0, "every K extent is whole 32-wide K-slabs; only layers 0 / 5 have tails");
__host__ __device__ constexpr uint32_t layer_bytes(int l) { return (uint32_t)num_halves(l) * layer_k(l) * 256u; }
__host__ __device__ constexpr uint32_t layer_offset(int l) {
  uint32_t o = 0;
  for (int i = 0; i < l; ++i) o += layer_bytes(i);
  return o;
}
// image offset of K-slab s of N-half h of layer l (its stages are contiguous in streaming order)
__host__ __device__ constexpr uint32_t w_stage_offset(bool wide, int l, int h, int s) {
  return layer_offset(l) + ((uint32_t)h * layer_k(l) + w_stage(wide, l, s).k0) * 256u;
}
// the producer streams the image front to back: stage after stage, in issue order, with no gaps
constexpr bool w_stages_contiguous(bool wide) {
  uint32_t o = 0;
  for (int l = 0; l < kNumLayers; ++l)
    for (int h = 0; h < num_halves(l); ++h)
      for (int s = 0; s < num_slabs(wide, l); ++s) {
        if (w_stage_offset(wide, l, h, s) != o) return false;
        o += w_stage(wide, l, s).bytes;
      }
  return o == layer_offset(kNumLayers);
}
static_assert(w_stages_contiguous(true) && w_stages_contiguous(false), "stage table and image layout disagree");
constexpr uint32_t kImageStageBytes = layer_offset(kNumLayers);
constexpr size_t kSmallOffset = ((size_t)kImageStageBytes + 255) / 256 * 256;
// view-direction part of the view layer, transposed for coalesced per-ray reads by the ray prologue:
// fp32 [27][128] weights W_view[n, 256 + k] as [k][n], then the 128 biases
constexpr size_t kViewDirOffset = kSmallOffset + ((sizeof(SmallParams) + 255) / 256 * 256);
constexpr size_t kViewDirBytes = (size_t)(kViewDim + 1) * kCond * sizeof(float);
constexpr size_t kImageBytes = kViewDirOffset + ((kViewDirBytes + 255) / 256 * 256);
// Split-operand ("x3") modes: a second stage image with the LOW halves of the weights (w - fl16(w), rounded to the
// same 16-bit format), same internal layout as the stage part of the first image, appended after it.
constexpr size_t kLoOffset = kImageBytes;
constexpr size_t kLoBytes = ((size_t)kImageStageBytes + 255) / 256 * 256;
constexpr size_t kImageEnd = kLoOffset + kLoBytes;

// Shapes below are for n = 128 samples per ray (kT = 1); a kT = 2 launch has n = 256: [B,257] fenceposts, [B,256]
// weights and density normals.  The training dump and MLP-only mode exist for kT = 1 only.
struct LevelParams {
  const uint8_t* wimage;
  const float* origins;
  const float* directions;
  const float* radii;
  float* t;                // [B,129] fenceposts of this level (read; written first when t_mode != 0)
  float* view_bias;        // [B,128]  b_view + W_view[:,256:] . pos_enc(viewdir) (written first when vb_mode != 0)
  // Ray prologue, run by the helper warps ahead of each ray's features: fenceposts / view bias produced in the level kernel
  // instead of by launches of their own.
  int t_mode;              // 0: read p.t; 1: coarse fenceposts from near/far (models/mip.py:143-160);
                           // 2: resample t_prev / w_prev (models/mip.py:232-280)
  int vb_mode;             // 0: read p.view_bias; 1: compute it from viewdirs and the fp32 view-layer weights
  const float* near;       // t_mode 1
  const float* far;
  Draws t_rand;            // t_mode 1, randomized: the [B,129] stratified uniforms (array or in-kernel Philox)
  int disparity;
  const float* t_prev;     // t_mode 2: previous level's fenceposts [B,129] and weights [B,128]
  const float* w_prev;
  Draws u_jitter;          // t_mode 2, randomized: the [B,129] inverse-CDF jitter (array or in-kernel Philox)
  int64_t* inds;           // t_mode 2: optional searchsorted indices [B,129]
  int randomized;
  float resample_padding;
  const float* viewdirs;   // vb_mode 1: [B,3]; the weights come from the packed image (kViewDirOffset)
  const float* feat_in;    // MLP-only mode (mipnerf_b200_mlp_forward): [B,128,96] features supplied by the caller
  float* raw_rgb_out;      // MLP-only mode: [B,128,3] / [B,128] raw heads instead of compositing
  float* raw_density_out;
  // Training forward: every activation the backward pass needs leaves the SM exactly as the tensor core saw it — the
  // 16-bit SW128 activation tile of each trunk layer / the bottleneck is stored from the epilogue's registers (bf16 /
  // fp16) or copied out of shared memory by bulk stores after its epilogue (split modes); the view layer's output and
  // the raw heads go out from registers.
  uint8_t* act_dump;       // [9][dump_tiles][64 KB]: h_0..h_7 (post-ReLU), bottleneck; tile = ray
  uint8_t* v_dump;         // [dump_tiles][32 KB]: view-layer output (post-ReLU), two SW128 slabs
  float* raw_rgb_keep;     // [B,128,3] / [B,128]: raw heads (before the activations) for render_backward
  float* raw_density_keep;
  int64_t dump_tiles;
  float* comp_rgb;
  float* distance;
  float* acc;
  float* weights;  // [B,128]
  int64_t num_rays;
  int white_bkgd;
  int disable_integration;
  float density_bias, rgb_scale, rgb_padding;
  Draws dnoise;  // density noise of randomized mode (models/mip_nerf.py:232-233): normals [B,128] or in-kernel; scale = std
  // Density-only mode (mipnerf_b200_query_density): tile i holds points 128 i .. 128 i + 127 of the Gaussians
  // q_means / q_covs [num_points, 3] (q_covs null: zero covariance); raw density into raw_density_out, softplus(raw +
  // density_bias) into density_out (either may be null).  num_rays counts the tiles.
  const float* q_means;
  const float* q_covs;
  int64_t num_points;
  float* density_out;
  // Radiance mode (mipnerf_b200_query_radiance): the query points as in density-only mode, each with its own direction
  // viewdirs [num_points, 3]; view_bias is the per-CTA slots [gridDim.x][2][128][128] of the points' view-direction
  // terms (tile parity); raw heads into raw_rgb_out / raw_density_out, their activations into rgb_out / density_out (any
  // may be null).
  float* rgb_out;
  // View-accumulator mode (mipnerf_b200_query_radiance_dirs): the query points as in density-only mode; the view layer's
  // pre-activation without its bias and view-direction columns, W_view[:, :256] . bottleneck, of every row of tile i
  // into view_acc + i [128][128] fp32 (rows past the last point hold garbage); densities as in density-only mode.
  float* view_acc;
};

// Compile-time modes of the level kernel: the forward (rays in, composited pixels out; MLP-only mode and the training
// forward are runtime variants of it), density-only queries, radiance queries with a view direction per point, and
// the view accumulators of radiance queries under a shared direction set.
enum LevelMode : int { kModeForward = 0, kModeDensity = 1, kModeRadiance = 2, kModeViewAcc = 3 };

// raw density of (ray, row) of a ray of kNs samples with the density noise added; kept out of line so that the
// (default) noise-free path carries none of the generator's registers
template <int kNs>
__device__ __noinline__ float noisy_raw_density(float raw, const Draws d, int64_t ray, int row) {
  return add_density_noise(raw, d, ray, row, kNs);
}

__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Phase accounting of the level kernel (tools/level_phases.py): built with -DMIPNERF_LEVEL_PHASES, thread 0 of each
// consumer warpgroup, the producer thread and the first helper thread charge the clock64 cycles since their previous
// mark to a phase, per CTA and per level (slot 0: coarse fenceposts, slot 1: resampled).  Without the define,
// PhaseClock is empty and every mark compiles to nothing.
enum LevelPhase : int {
  kPhPrologue,   // helpers: fenceposts / resampler, view bias
  kPhIpe,        // helpers: Gaussians + IPE features
  kPhWFull,      // consumers: waiting for a weight stage (w_full)
  kPhMma,        // consumers: wgmma issue and retire
  kPhEpilogue,   // layer epilogue chunks (their K-slab's wgmmas run meanwhile), view layer + colour head, head
                 // reductions, activation-dump stores
  kPhComposite,  // helpers: activations + compositing (or the raw heads of MLP-only mode)
  kPhBarrier,    // named-barrier waits (bf16 / fp16 consumers: none inside the layer loop), consumers' heads_empty
  kPhWEmpty,     // producer: waiting for a free ring slot (w_empty)
  kPhIssue,      // producer: everything else
  kPhFeatFull,   // consumers: waiting for the ray's feature buffer (feat_full)
  kPhFeatEmpty,  // helpers: waiting for a free feature buffer (feat_empty)
  kPhHeadsFull,  // helpers: waiting for the raw heads of the ray to composite (heads_full)
  kPhTotal,      // clock64 cycles from the role's first mark to its last
  kNumPhases
};
#ifdef MIPNERF_LEVEL_PHASES
constexpr int kNumRoles = 4;  // consumer warpgroup 0, consumer warpgroup 1, weight producer, helpers
constexpr int kPhaseMaxCtas = 1024;
constexpr uint32_t kPhaseBytes = kNumRoles * kNumPhases * 8;  // shared-memory accumulators, one row per role
// [slot][cta][role][phase]
__device__ unsigned long long g_level_phases[2][kPhaseMaxCtas][kNumRoles][kNumPhases];
struct PhaseClock {
  unsigned long long* acc;  // this role's row in shared memory; null on the threads that do not measure
  long long start, last;
  __device__ __forceinline__ void begin(unsigned long long* row, bool measuring) {
    acc = measuring ? row : nullptr;
    if (acc)
      for (int i = 0; i < kNumPhases; ++i) acc[i] = 0;
    start = last = clock64();
  }
  __device__ __forceinline__ void mark(int ph) {
    const long long now = clock64();
    if (acc) acc[ph] += (unsigned long long)(now - last);
    last = now;
  }
  __device__ __forceinline__ void end(int slot, int role) {
    if (!acc || blockIdx.x >= kPhaseMaxCtas) return;
    acc[kPhTotal] = (unsigned long long)(last - start);
    for (int i = 0; i < kNumPhases; ++i) atomicAdd(&g_level_phases[slot][blockIdx.x][role][i], acc[i]);
  }
};
#else
constexpr uint32_t kPhaseBytes = 0;
struct PhaseClock {
  __device__ __forceinline__ void begin(unsigned long long*, bool) {}
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void end(int, int) {}
};
#endif

template <int kFmt>
__device__ __forceinline__ void store8(uint8_t* dst, const float (&x)[8]) {
  *reinterpret_cast<uint4*>(dst) = make_uint4(pack2<kFmt>(x[0], x[1]), pack2<kFmt>(x[2], x[3]),
                                              pack2<kFmt>(x[4], x[5]), pack2<kFmt>(x[6], x[7]));
}

template <int kFmt>
__device__ __forceinline__ float2 unpack2(uint32_t v) {
  if (kFmt == 1) return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&v));
  return __half22float2(*reinterpret_cast<__half2*>(&v));
}
// x = hi + lo with hi = fl16(x), lo = fl16(x - hi): the two 16-bit operands of the split ("x3") modes
template <int kFmt>
__device__ __forceinline__ void store8_split(uint8_t* dst_hi, uint8_t* dst_lo, const float (&x)[8]) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    h[e] = pack2<kFmt>(x[2 * e], x[2 * e + 1]);
    const float2 f = unpack2<kFmt>(h[e]);
    l[e] = pack2<kFmt>(x[2 * e] - f.x, x[2 * e + 1] - f.y);
  }
  *reinterpret_cast<uint4*>(dst_hi) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(dst_lo) = make_uint4(l[0], l[1], l[2], l[3]);
}

// Gaussian + IPE features [8 gi_begin, 8 gi_end) and [48 + 8 gi_begin, 48 + 8 gi_end) of one sample row of a ray (or,
// in MLP-only mode, the caller's features) into the feature tile: SW128 slab (K 0..63) + SW64 tail (K 64..95).  `row`
// is the row of the tile; MLP-only mode has one tile per ray.  kDensity (the query modes, density and radiance): the
// row is query point 128 ray + row (zero past the last one), encoded with the IPE of mipnerf_b200_integrated_pos_enc
// (ipe_pair<false>), so that the 16-bit features equal MLP-only mode's rounding of that entry point's output.
template <int kFmt, bool kX3, int kT, bool kDensity = false>
__device__ __forceinline__ void ipe_row_group(const LevelParams& p, const RayGeom& g, int64_t ray, int row, float t0,
                                              float t1, uint8_t* myF, int gi_begin, int gi_end) {
  float mean[3] = {0.f, 0.f, 0.f}, cov[3] = {0.f, 0.f, 0.f};
  const float* fin = nullptr;
  if (kDensity) {
    const int64_t pt = ray * kN + row;
    if (pt < p.num_points) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        mean[c] = __ldg(p.q_means + pt * 3 + c);
        cov[c] = p.q_covs && !p.disable_integration ? __ldg(p.q_covs + pt * 3 + c) : 0.f;
      }
    }
  } else if (kT == 1 && p.feat_in) {
    fin = p.feat_in + (ray * kN + row) * kFeat;  // MLP-only mode: the caller's encoding
  } else {
    float tm, tv, rv;
    frustum_moments(t0, t1, g.radius_sq, tm, tv, rv);
    lift_gaussian(g, tm, tv, rv, mean, cov);
    if (p.disable_integration) cov[0] = cov[1] = cov[2] = 0.f;
  }
#pragma unroll
  for (int gi = 0; gi < 6; ++gi) {
    if (gi < gi_begin || gi >= gi_end) continue;
    float fsin[8], fcos[8];
    if (fin) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        fsin[e] = __ldg(fin + gi * 8 + e);
        fcos[e] = __ldg(fin + 48 + gi * 8 + e);
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int f = gi * 8 + e;  // feature index = degree*3 + coord   (models/mip.py:335-341)
        // (measured: the accurate sinf / expf in place of the MUFU pair changes the split modes' error against the
        //  reference goldens by < 3 % — 1.06e-4 vs 1.08e-4 on the worst one — and costs 7x the IPE time: not used)
        ipe_pair<!kDensity>(mean[f % 3], cov[f % 3], f / 3, fsin[e], fcos[e]);
      }
    }
    const uint32_t o_sin = sw128_offset(row, gi * 8);                                     // K = f
    const uint32_t o_cos = gi < 2 ? sw128_offset(row, 48 + gi * 8)                        // K = 48 + f < 64
                                  : kStageBytes + sw64_offset(row, (gi - 2) * 8);         // K = 64.. -> SW64 tail
    if (kX3) {  // low halves go to the second feature tile
      store8_split<kFmt>(myF + o_sin, myF + kFBytes + o_sin, fsin);
      store8_split<kFmt>(myF + o_cos, myF + kFBytes + o_cos, fcos);
    } else {
      store8<kFmt>(myF + o_sin, fsin);
      store8<kFmt>(myF + o_cos, fcos);
    }
  }
}

// =================================================================================================
// The level kernel (sm_90a): one persistent CTA per SM, 384 threads, one tile of 128 sample rows at a time in the
// tensor core, with the scalar work of the neighbouring tiles beside it.  A ray is kT = 1 or 2 consecutive tiles
// (128 or 256 samples); below, "ray" is a tile when kT = 2, except for the per-ray prologue and compositing.
//   * warps 0-3 / 4-7: two consumer warpgroups, warpgroup g owns sample rows 64 g .. 64 g + 63 of the ray.  Each
//     issues the wgmma (M = 64, N = 128, K = 16) of every layer for its rows (A operand: its rows of the ray's feature
//     buffer in shared memory for layer 0 and layer 5's skip slabs; otherwise the layer input in registers (bf16 /
//     fp16) or its rows of the activation tile in shared memory (split modes); B: the weight stage both warpgroups
//     share), runs the epilogue from the register accumulators straight into the next layer's A operand in chunks
//     under the wgmmas of later K-slabs (software-pipelined layer loop), and leaves the raw heads of its rows in shared
//     memory.  The rows of a warpgroup are private to it, so a layer boundary is at most a 128-thread barrier.
//   * warps 8-11: producer warpgroup (setmaxnreg gives registers to the consumers).  Warp 8 is the weight producer
//     — cp.async.bulk of the pre-swizzled weight stages of the packed image (w_stage; + the low-half stage in the
//     split modes) into a ring of 16 KB slots; a slot is free once both warpgroups' wgmmas reading it have completed.
//   * warps 9-11 are the helpers: while the consumers run the layers of ray r, they run the ray prologue of ray r + 1
//     (the coarse fenceposts (level 0) or the bit-exact inverse-CDF resampler (levels >= 1), and the per-ray
//     view-layer bias (level 0; later levels read it back), which they leave in a shared-memory slot for the view
//     layer's epilogue), write its Gaussians + IPE features into a free feature buffer, and then composite ray r once
//     its raw heads are in.
// Hand-offs (mbarriers): feat_full[b] (helpers -> consumers: the features of buffer b are written and fenced for the
// async proxy), feat_empty[b] (consumers -> helpers: the wait that retires layer 5's last skip K-slab has returned, the
// last read of the buffer), heads_full[par] / heads_empty[par] (the raw heads of rays of parity par).  A forward is one
// launch of this kernel per level and nothing else.  The layer-5 skip connection is three extra K slabs read from the
// feature buffer (no concat).
// =================================================================================================
// 384 threads = three warpgroups; the producer warpgroup hands its registers to the consumers (setmaxnreg): 2 x 128 x
// kConsumerRegs + 128 x kProducerRegs fill the register file, and the consumers' two live N = 128 accumulators fit
// without spills.
constexpr int kThreads = 384;
constexpr int kHelperWarp0 = 9;  // warps 9-11
constexpr int kHelperThreads = 96;
constexpr int kHelperBar = 3;  // named barrier of the helper warps (1 and 2: the consumer warpgroups' own)
constexpr int kHeadsWriters = 2 * 128 / 4;  // one consumer thread per quad stores the raw heads of its two rows
#ifndef MIPNERF_LEVEL_PRODUCER_REGS
#define MIPNERF_LEVEL_PRODUCER_REGS 40
#endif
constexpr int kProducerRegs = MIPNERF_LEVEL_PRODUCER_REGS;
constexpr int kConsumerRegs = (65536 / 128 - kProducerRegs) / 2 / 8 * 8;
static_assert(2 * 128 * kConsumerRegs + 128 * kProducerRegs <= 65536 && kProducerRegs % 8 == 0, "setmaxnreg split");
// Weight-ring depth of the bf16 / fp16 kernel in 16 KB slots (a -D flag overrides it for experiments).
#ifndef MIPNERF_LEVEL_STAGES
#define MIPNERF_LEVEL_STAGES 6
#endif
template <bool kX3, int kT>
struct LevelLayout {
  // Feature buffers, one tile each: bf16 / fp16 have two, so that the helpers write tile i + 1's features while layer
  // 0 / layer 5 of tile i read the other; the split modes (hi + lo tiles next to the 128 KB activation tile) have room
  // for one only, and the helpers write the next tile's features once layer 5's skip slabs have retired.
  static constexpr int kFeatBufs = kX3 ? 1 : 2;
  static constexpr uint32_t kFBuf = (kX3 ? 2 : 1) * kFBytes;  // one buffer: the feature tile (split modes: hi, lo)
  // bf16 / fp16: the layer inputs live in registers, so the CTA holds only the feature buffers and the weight ring, and
  // the ring is as deep as the 164 KB carveout allows: 6 slots (96 KB).
  static constexpr int kStages = kX3 ? 2 : MIPNERF_LEVEL_STAGES;
  // a ring slot: one wide stage (or a tail), or the W_hi then W_lo stage of a split-mode K-slab
  static constexpr uint32_t kStage = 16384;
  static constexpr uint32_t kA = 0;  // split modes only: the activation tile, hi then lo
  static constexpr uint32_t kF = kA + (kX3 ? 2 * kABytes : 0);
  static constexpr uint32_t kW = kF + kFeatBufs * kFBuf;
  static constexpr uint32_t kMisc = kW + kStages * kStage;
  // mbarriers: w_full / w_empty [kStages], feat_full / feat_empty [kFeatBufs], heads_full / heads_empty [2]
  static constexpr int kNumMbars = 2 * kStages + 2 * kFeatBufs + 2 * 2;
  // mbarriers, raw heads [2][128][4] (tile parity; with kT = 2 the two tiles of a ray), scan carries [4 kT], partial
  // sums [4 kT][8] (one per 32-row chunk of the ray), resampler scratch [128 kT + 1]
  static constexpr uint32_t kMiscBytes =
      kNumMbars * 8 + 2 * kN * 4 * 4 + 4 * kT * 4 + 4 * kT * 8 * 4 + (kT * kN + 1) * 4;
  // the forward's per-ray view bias [2][128] fp32 (parity of the ray's index in the CTA): the helpers fill it in the
  // ray prologue, the consumers' view-layer epilogue reads it
  static constexpr uint32_t kVBias = (kMisc + kMiscBytes + 15) & ~15u;
  static constexpr uint32_t kVBiasBytes = 2 * kCond * 4;
  static constexpr uint32_t kPhase = kVBias + kVBiasBytes;  // phase accumulators (MIPNERF_LEVEL_PHASES)
  // + slack for the 1024-B alignment of the tiles
  static constexpr uint32_t kTotal = kPhase + kPhaseBytes + 1024;
  static_assert(kT == 1 || kT == 2, "a ray is one or two 128-row tiles");
  static_assert(kNumMbars % 2 == 0, "the raw heads behind the mbarriers must be 16-B aligned");
  static_assert(kTotal <= 232448, "exceeds 227 KB of shared memory per CTA");
  static_assert(kX3 || kStages * kStage > 72 * 1024 || kTotal + 1024 <= 132 * 1024,
                "bf16 / fp16 with a weight ring of up to 72 KB no longer fits the 132 KB carveout");
  static_assert(kX3 || kStages * kStage > 96 * 1024 || kTotal + 1024 <= 164 * 1024,
                "bf16 / fp16 with a weight ring of up to 96 KB no longer fits the 164 KB carveout");
  static_assert(kX3 ? kStage == 2 * w_stage(false, 0, 0).bytes : kStage == w_stage(true, 1, 0).bytes,
                "a ring slot holds one stage (split modes: its hi and lo stages)");
};

// does column k of layer l's input come from the feature tile (layer 0, layer 5's skip columns)?
__device__ __forceinline__ bool level_reads_feat(int l, int k) { return l == 0 || (l == 5 && k >= kWidth); }
// A-operand descriptor of the K step (16 wide) at column k of layer l, for the rows of one warpgroup: the activation
// tile (split modes), or the feature tile's SW128 slab (K 0..63) and SW64 tail (K 64..95)
__device__ __forceinline__ uint64_t level_a_desc(int l, int k, uint32_t a_u, uint32_t f_u, uint32_t ft_u) {
  if (!level_reads_feat(l, k)) return make_sw128_desc(a_u + (uint32_t)(k >> 6) * kStageBytes + 2u * (uint32_t)(k & 63));
  const int kf = l == 0 ? k : k - kWidth;
  if (kf < 64) return make_sw128_desc(f_u + 2u * (uint32_t)kf);
  return make_sw64_desc(ft_u + 2u * (uint32_t)(kf - 64));
}

// Where a consumer warpgroup stands in the weight ring: the slot and phase of its next stage, and the slot of its newest
// wgmma group (-1: none in flight).
struct RingPos {
  int st;
  uint32_t ph;
  int prev;
};

// K-slab s (w_stage) of one N = 128 half of layer l into acc, for the rows of one warpgroup: wait for the weight stage,
// issue its wgmmas as one group, then wait until only that group is in flight.  The wait retires the previous group,
// whose stage is released (one arrive per warpgroup); so one stage's wgmmas stay in flight across calls, also from one
// half or layer to the next.
template <bool kX3>
__device__ __forceinline__ uint32_t level_stage_acquire(uint32_t w_u, uint64_t* w_full, const RingPos& rp,
                                                        PhaseClock& clk) {
  mbar_wait(&w_full[rp.st], rp.ph);
  clk.mark(kPhWFull);
  wgmma_fence();
  return w_u + (uint32_t)rp.st * LevelLayout<kX3, 1>::kStage;
}
template <bool kX3>
__device__ __forceinline__ void level_stage_commit(uint64_t* w_empty, RingPos& rp, bool leader, PhaseClock& clk) {
  wgmma_commit();
  wgmma_wait<1>();
  if (rp.prev >= 0 && leader) mbar_arrive(&w_empty[rp.prev]);
  rp.prev = rp.st;
  if (++rp.st == LevelLayout<kX3, 1>::kStages) {
    rp.st = 0;
    rp.ph ^= 1;
  }
  clk.mark(kPhMma);
}
template <int kFmt, bool kX3>
__device__ __forceinline__ void level_mma_slab(float (&acc)[64], int l, int s, uint32_t a_u, uint32_t f_u,
                                               uint32_t ft_u, uint32_t w_u, uint64_t* w_full, uint64_t* w_empty,
                                               RingPos& rp, bool leader, PhaseClock& clk) {
  const uint32_t b_u = level_stage_acquire<kX3>(w_u, w_full, rp, clk);
  const WStage ws = w_stage(!kX3, l, s);  // bf16 / fp16: l and s are compile-time constants here
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (16 * j >= ws.kw) break;
    const uint64_t a_hi = level_a_desc(l, ws.k0 + 16 * j, a_u, f_u, ft_u);
    const uint64_t b_hi = ws.sw128 ? make_sw128_desc(b_u + 32u * j) : make_sw64_desc(b_u + 32u * j);
    wgmma_m64n128k16<kFmt>(acc, a_hi, b_hi, (s | j) ? 1u : 0u);
    if (kX3) {  // A_lo . W_hi + A_hi . W_lo (the lo tiles sit one tile size behind the hi tiles)
      wgmma_m64n128k16<kFmt>(acc, a_hi + (level_reads_feat(l, ws.k0) ? kFBytes : kABytes) / 16, b_hi, 1u);
      wgmma_m64n128k16<kFmt>(acc, a_hi, b_hi + ws.bytes / 16, 1u);
    }
  }
  level_stage_commit<kX3>(w_empty, rp, leader, clk);
}
// The same for the 64-wide K-slab s < 4 of layers 1..9 in the bf16 / fp16 kernel, with A from registers: x is the layer
// input as wgmma A fragments (see level_epilogue_chunk_rs), and K-slab s reads x[16 s .. 16 s + 15].  `s` must be a
// compile-time constant after unrolling, so that x stays in registers.
template <int kFmt>
__device__ __forceinline__ void level_mma_slab_rs(float (&acc)[64], const uint32_t (&x)[64], int s, uint32_t w_u,
                                                  uint64_t* w_full, uint64_t* w_empty, RingPos& rp, bool leader,
                                                  PhaseClock& clk) {
  const uint32_t b_u = level_stage_acquire<false>(w_u, w_full, rp, clk);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t a[4] = {x[16 * s + 4 * j], x[16 * s + 4 * j + 1], x[16 * s + 4 * j + 2], x[16 * s + 4 * j + 3]};
    wgmma_m64n128k16_rs<kFmt>(acc, a, make_sw128_desc(b_u + 32u * j), (s | j) ? 1u : 0u);
  }
  level_stage_commit<false>(w_empty, rp, leader, clk);
}

// The layer epilogues run in chunks under the wgmmas of K-slabs (see the layer loop of mlp_level_kernel): kEpiChunks
// chunks per N = 128 half, each after the wait of a K-slab; chunk c covers the accumulator's column groups
// 4 c .. 4 c + 3, i.e. columns c_base + 32 c .. + 31, which are exactly the A-operand columns that the 32-wide
// K-slab c (c_base = 0) or 4 + c (c_base = 128) of the next layer reads in the split modes.
constexpr int kEpiChunks = 4;
constexpr int kEpiGroups = 16 / kEpiChunks;
// First K-slab of a trunk layer's N-half 1 that carries a chunk of N-half 0's epilogue (chunk c after K-slab
// kEpiOverlap + c).  Any value in 1..4 is safe: chunk c overwrites the columns of K-slab c, retired by then.  Measured
// on an H100 80GB HBM3 at 400 W (bench.py bf16 step, before the bias loads moved ahead of the K-slab): 4.13-4.15 ms
// with 1, 4.22 / 4.35 / 4.48 ms with 2 / 3 / 4.
constexpr int kEpiOverlap = 1;
static_assert(kEpiOverlap >= 1 && kEpiOverlap + kEpiChunks <= 8, "chunk c must follow the retirement of K-slab c");

// The bias of one epilogue chunk, loaded before the K-slab that the chunk follows, so that the load latency hides
// under that slab's wgmmas.
struct EpiConsts {
  float2 b[kEpiGroups];
};
__device__ __forceinline__ void level_epilogue_consts(EpiConsts& e, int l, int c_base, int chunk, int cq,
                                                      const SmallParams* __restrict__ gsp) {
#pragma unroll
  for (int jj = 0; jj < kEpiGroups; ++jj)
    e.b[jj] = __ldg(reinterpret_cast<const float2*>(gsp->bias[l] + c_base + 8 * (kEpiGroups * chunk + jj) + cq));
}

// Epilogue chunk `chunk` of one N = 128 half (columns c_base..) of trunk layer / bottleneck l: + bias -> ReLU (l < 8)
// -> 16-bit -> the A operand of the next layer (rows r0, r0 + 8 of the fragment); l == 7 also accumulates the density
// head on the fp32 (un-rounded) h7 (models/mip_nerf.py:98).  `chunk` must be a compile-time constant after unrolling,
// so that the accumulator stays in registers.
template <int kFmt, bool kX3>
__device__ __forceinline__ void level_epilogue_chunk(const float (&acc)[64], const EpiConsts& e, int l, int c_base,
                                                     int chunk, int r0, int cq, uint8_t* sA,
                                                     const SmallParams* __restrict__ gsp, float& d0, float& d1) {
  const bool relu = l < 8;
  // sw128_offset(r0, c & 63) = row_off | ((j & 7) << 4 ^ sw): one LOP3 per store.  Opaque per chunk, so that the
  // compiler recomputes the offsets instead of computing them once and keeping them in local memory across the layers.
  uint32_t row_off = (uint32_t)r0 * 128u + 2u * (uint32_t)cq, sw = (uint32_t)(r0 & 7) << 4;
  asm volatile("" : "+r"(row_off), "+r"(sw));
#pragma unroll
  for (int jj = 0; jj < kEpiGroups; ++jj) {
    const int j = kEpiGroups * chunk + jj;
    const float2 b = e.b[jj];
    float a0 = acc[4 * j], a1 = acc[4 * j + 1], a2 = acc[4 * j + 2], a3 = acc[4 * j + 3];
    fadd2(a0, a1, b.x, b.y);
    fadd2(a2, a3, b.x, b.y);
    if (l == 7) {
      const float2 wd = __ldg(reinterpret_cast<const float2*>(gsp->w_density + c_base + 8 * j + cq));
      ffma2(d0, d1, fmaxf(a0, 0.f), fmaxf(a2, 0.f), wd.x, wd.x);
      ffma2(d0, d1, fmaxf(a1, 0.f), fmaxf(a3, 0.f), wd.y, wd.y);
    }
    if (relu) a0 = fmaxf(a0, 0.f), a1 = fmaxf(a1, 0.f), a2 = fmaxf(a2, 0.f), a3 = fmaxf(a3, 0.f);
    const uint32_t o0 = (uint32_t)((c_base >> 6) + (j >> 3)) * kStageBytes + (row_off | ((uint32_t)(j & 7) << 4 ^ sw));
    const uint32_t o1 = o0 + 8u * 128u;  // row r0 + 8: same swizzle phase
    const uint32_t h0 = pack2<kFmt>(a0, a1), h1 = pack2<kFmt>(a2, a3);
    *reinterpret_cast<uint32_t*>(sA + o0) = h0;
    *reinterpret_cast<uint32_t*>(sA + o1) = h1;
    if (kX3) {  // hi = fl16(x), lo = fl16(x - hi): 22 (fp16) / 16 (bf16) significant bits reach the next layer
      const float2 f0 = unpack2<kFmt>(h0), f1 = unpack2<kFmt>(h1);
      *reinterpret_cast<uint32_t*>(sA + kABytes + o0) = pack2<kFmt>(a0 - f0.x, a1 - f0.y);
      *reinterpret_cast<uint32_t*>(sA + kABytes + o1) = pack2<kFmt>(a2 - f1.x, a3 - f1.y);
    }
  }
}

// ---- the register-chained layer loop of the bf16 / fp16 kernel (64-wide K-slabs) ----
// Where acc0's epilogue chunks run under a layer's N-half 1, counted in 32-wide halves of its K-slabs: chunk c follows
// the K-slab (kEpiFirstRs + c) / 2.  The default 4 puts chunks 0, 1 after K-slab 2 and chunks 2, 3 after K-slab 3.
// The chunks write registers that no wgmma in flight reads, and the wait of N-half 1's first K-slab retires all of
// N-half 0, so any value in 0..4 is safe; a -D flag overrides it for experiments.  0 and 1 make ptxas serialise the
// wgmmas (too few registers); 2 and 3 leave a local-memory load in the layer loop.  Measured with bench.py (bf16 step,
// 6 slots, H100 80GB HBM3 at 400 W): 2.86-2.88 ms with 2, 2.84 ms with 3, 2.83-2.85 ms with 4.
#ifndef MIPNERF_LEVEL_EPI_FIRST
#define MIPNERF_LEVEL_EPI_FIRST 4
#endif
constexpr int kEpiFirstRs = MIPNERF_LEVEL_EPI_FIRST;
static_assert(kEpiFirstRs >= 0 && kEpiFirstRs + kEpiChunks <= 8, "the chunks must follow K-slabs 0..3");
__host__ __device__ constexpr int epi_slab_acc0(int c) { return (kEpiFirstRs + c) / 2; }
// acc1's chunks c = 0..3 follow the next layer's N-half-0 K-slab c / 2: chunk c writes x[32 + 8 c .. 32 + 8 c + 7],
// which K-slab 2 (chunks 0, 1) and K-slab 3 (chunks 2, 3) read, and the wait of K-slab 0 retires all of the layer.
__host__ __device__ constexpr int epi_slab_acc1(int c) { return c / 2; }
static_assert(epi_slab_acc1(kEpiChunks - 1) < 2, "acc1's chunks must land before the next layer's K-slab 2 reads them");

// What the layer loop needs besides its accumulators and A arrays.
struct LevelRsCtx {
  uint32_t f_u, ft_u, w_u;  // this warpgroup's rows of the ray's feature buffer (SW128 slab, SW64 tail), the weight ring
  uint64_t* w_full;
  uint64_t* w_empty;
  uint64_t* feat_empty;    // the ray's feature buffer is free once layer 5's skip slabs have retired
  const SmallParams* gsp;
  uint8_t* dump;           // training forward: this ray's tile of h_0 in p.act_dump (h_l: + l dump_stride); else null
  size_t dump_stride;
  uint64_t dump_policy;
  int r0, cq;
  bool leader;
};

// Epilogue chunk of the bf16 / fp16 kernel: the arithmetic of level_epilogue_chunk, with the 16-bit pairs kept in
// registers as the next layer's wgmma A fragments instead of stored to shared memory.  The accumulator fragment of
// column group j (columns 8 j + cq, + 1 of rows r0 and r0 + 8, j counted over all 256 columns) is half of the A
// fragment of K-step j / 2: x[2 j] holds row r0, x[2 j + 1] row r0 + 8.  In the training forward the same pairs also
// go to the layer's activation tile in global memory, at their SW128 tile-image offsets.
template <int kFmt>
__device__ __forceinline__ void level_epilogue_chunk_rs(const float (&acc)[64], const EpiConsts& e, int l, int c_base,
                                                        int chunk, uint32_t (&x)[64], const LevelRsCtx& k, float& d0,
                                                        float& d1) {
  const bool relu = l < 8;
  uint8_t* dump = k.dump ? k.dump + (size_t)l * k.dump_stride : nullptr;
#pragma unroll
  for (int jj = 0; jj < kEpiGroups; ++jj) {
    const int j = kEpiGroups * chunk + jj;
    const float2 b = e.b[jj];
    float a0 = acc[4 * j], a1 = acc[4 * j + 1], a2 = acc[4 * j + 2], a3 = acc[4 * j + 3];
    fadd2(a0, a1, b.x, b.y);
    fadd2(a2, a3, b.x, b.y);
    if (l == 7) {
      const float2 wd = __ldg(reinterpret_cast<const float2*>(k.gsp->w_density + c_base + 8 * j + k.cq));
      ffma2(d0, d1, fmaxf(a0, 0.f), fmaxf(a2, 0.f), wd.x, wd.x);
      ffma2(d0, d1, fmaxf(a1, 0.f), fmaxf(a3, 0.f), wd.y, wd.y);
    }
    // ReLU in the conversion (F2FP.RELU): rounding keeps the sign, so clamping after it gives max(x, 0) rounded, the
    // same bits as fmaxf then pack2 for every x but NaN (which fmaxf would turn into 0)
    const int jg = (c_base >> 3) + j;
    x[2 * jg] = relu ? pack2_relu<kFmt>(a0, a1) : pack2<kFmt>(a0, a1);
    x[2 * jg + 1] = relu ? pack2_relu<kFmt>(a2, a3) : pack2<kFmt>(a2, a3);
  }
  if (dump) {
    // The four threads of a quad hold the four 4-byte quarters of the chunk's four 16-byte column groups (per row): a
    // 4 x 4 transpose in the quad (two butterfly steps) gives thread q all of group 4 chunk + q, one 16-byte store per
    // row, so that every store fills whole L2 sectors.
    const int q = k.cq >> 1;
    const int jg = (c_base >> 3) + kEpiGroups * chunk + q;
    const uint32_t o0 = (uint32_t)(jg >> 3) * kStageBytes + sw128_offset(k.r0, 8 * (jg & 7));
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // row r0, row r0 + 8
      uint32_t v[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) v[jj] = x[2 * ((c_base >> 3) + kEpiGroups * chunk + jj) + h];
#pragma unroll
      for (int i = 0; i < 2; ++i) {  // exchange the 2 x 2 blocks off the diagonal with quad thread q ^ 2
        const uint32_t r = __shfl_xor_sync(0xffffffffu, (q & 2) ? v[i] : v[2 + i], 2);
        if (q & 2) v[i] = r;
        else v[2 + i] = r;
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {  // then the elements off the diagonal of each block with quad thread q ^ 1
        const uint32_t r = __shfl_xor_sync(0xffffffffu, (q & 1) ? v[2 * i] : v[2 * i + 1], 1);
        if (q & 1) v[2 * i] = r;
        else v[2 * i + 1] = r;
      }
      st_global_v4_hint(dump + o0 + (uint32_t)h * 8u * 128u, make_uint4(v[0], v[1], v[2], v[3]), k.dump_policy);
    }
  }
}

// Layer l + 1's N-half 0, K-slabs 0, 1 (x[0..31], from acc0's epilogue of layer l) into acc0, with acc1's epilogue of
// layer l (x[32..63]) in chunks after them (epi_slab_acc1).  The wait of the first K-slab retires all of layer l; after
// layer 5 (release_feat) that is the last read of the feature buffer, which goes back to the helpers.
template <int kFmt>
__device__ __forceinline__ void level_rs_next_head(float (&acc0)[64], float (&acc1)[64], uint32_t (&x)[64], int l,
                                                   bool release_feat, const LevelRsCtx& k, RingPos& rp, PhaseClock& clk,
                                                   float& d0, float& d1) {
  wgmma_fence_acc(acc0);
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    EpiConsts e[kEpiChunks];
#pragma unroll
    for (int c = 0; c < kEpiChunks; ++c)
      if (epi_slab_acc1(c) == s) level_epilogue_consts(e[c], l, 128, c, k.cq, k.gsp);
    level_mma_slab_rs<kFmt>(acc0, x, s, k.w_u, k.w_full, k.w_empty, rp, k.leader, clk);
    if (s == 0 && release_feat && k.leader) mbar_arrive(k.feat_empty);
    if (s == 0) wgmma_fence_acc(acc1);
#pragma unroll
    for (int c = 0; c < kEpiChunks; ++c)
      if (epi_slab_acc1(c) == s) level_epilogue_chunk_rs<kFmt>(acc1, e[c], l, 128, c, x, k, d0, d1);
    clk.mark(kPhEpilogue);
  }
}

// Trunk layer / bottleneck l (1..8) from x_in into x_out: the rest of N-half 0 into acc0, N-half 1 into acc1 with
// acc0's epilogue in chunks under it (epi_slab_acc0), then level_rs_next_head.  kSkip: l may be 5, whose K-slabs 4
// (SW128) and 5 (SW64 tail) read the feature tile.  kLast (density-only mode, l = 7): no next layer; the wgmmas retire
// and acc1's epilogue chunks follow in the order level_rs_next_head runs them, so the density head sums the same terms
// in the same order.
template <int kFmt, bool kSkip, bool kLast = false>
__device__ __forceinline__ void level_rs_layer(float (&acc0)[64], float (&acc1)[64], const uint32_t (&x_in)[64],
                                               uint32_t (&x_out)[64], int l, const LevelRsCtx& k, RingPos& rp,
                                               PhaseClock& clk, float& d0, float& d1) {
  const bool skip = kSkip && l == 5;
  // the feature tile's addresses, opaque here so that the compiler recomputes the skip slabs' descriptors instead of
  // keeping them in local memory across the layers
  uint32_t f_u = k.f_u, ft_u = k.ft_u;
  asm volatile("" : "+r"(f_u), "+r"(ft_u));
#pragma unroll
  for (int s = 2; s < kWidth / 64; ++s)
    level_mma_slab_rs<kFmt>(acc0, x_in, s, k.w_u, k.w_full, k.w_empty, rp, k.leader, clk);
  if (skip) {
#pragma unroll
    for (int s = kWidth / 64; s < num_slabs(true, 5); ++s)
      level_mma_slab<kFmt, false>(acc0, 5, s, 0u, f_u, ft_u, k.w_u, k.w_full, k.w_empty, rp, k.leader, clk);
  }
  wgmma_fence_acc(acc1);
#pragma unroll
  for (int s = 0; s < kWidth / 64; ++s) {
    EpiConsts e[kEpiChunks];  // the biases of the chunks that follow K-slab s, loaded before it
#pragma unroll
    for (int c = 0; c < kEpiChunks; ++c)
      if (epi_slab_acc0(c) == s) level_epilogue_consts(e[c], l, 0, c, k.cq, k.gsp);
    level_mma_slab_rs<kFmt>(acc1, x_in, s, k.w_u, k.w_full, k.w_empty, rp, k.leader, clk);
    if (s == epi_slab_acc0(0)) wgmma_fence_acc(acc0);
#pragma unroll
    for (int c = 0; c < kEpiChunks; ++c)
      if (epi_slab_acc0(c) == s) level_epilogue_chunk_rs<kFmt>(acc0, e[c], l, 0, c, x_out, k, d0, d1);
    clk.mark(kPhEpilogue);
  }
  if (skip) {
#pragma unroll
    for (int s = kWidth / 64; s < num_slabs(true, 5); ++s)
      level_mma_slab<kFmt, false>(acc1, 5, s, 0u, f_u, ft_u, k.w_u, k.w_full, k.w_empty, rp, k.leader, clk);
  }
  if constexpr (kLast) {
    wgmma_wait<0>();
    wgmma_fence_acc(acc1);
    if (k.leader) mbar_arrive(&k.w_empty[rp.prev]);
    rp.prev = -1;
    clk.mark(kPhMma);
#pragma unroll
    for (int c = 0; c < kEpiChunks; ++c) {
      EpiConsts e;
      level_epilogue_consts(e, l, 128, c, k.cq, k.gsp);
      level_epilogue_chunk_rs<kFmt>(acc1, e, l, 128, c, x_out, k, d0, d1);
    }
    clk.mark(kPhEpilogue);
  } else {
    level_rs_next_head<kFmt>(acc0, acc1, x_out, l, skip, k, rp, clk, d0, d1);
  }
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Radiance mode: the view-direction term  b_view[n] + W_view[n, 256:283] . pos_enc(viewdir)  of each query point of
// `tile` into its row of `slot` [128][128] (models/mip.py:353-363, models/mip_nerf.py:106-108).  fp32, with the
// encoding and the fmaf order (the bias, then k = 0..26) of the level-0 prologue and view_bias_from_enc_kernel, so that
// every term is theirs bit for bit.  A helper warp takes kViewPts points at a time: lane f < 27 encodes element f of
// each, and the lane owns outputs n = 4 lane .. 4 lane + 3, whose weights it loads once per k for all kViewPts points.
// Rows past the last point get the bias alone.  The stores go to L2 (st.cg); the consumers read them back with ld.cg
// after feat_full, as the forward's view bias.
constexpr int kViewPts = 4;
// Element f < 3 + 6 num_deg of the view encoding of direction vd (models/mip.py:353-363, append_identity): vd, then
// sin(2^l vd) scale-major then xyz, then sin(2^l vd + pi/2); the arithmetic of pos_enc_kernel, of level_view_terms and
// of the level-0 prologue.  (Those two keep their own copy of it: calling this function from them reorders their SASS.)
__device__ __forceinline__ float view_enc_elem(const float* vd, int f, int num_deg) {
  float enc;
  if (f < 3) {
    enc = __ldg(vd + f);  // append_identity
  } else {
    const int gidx = f - 3, half = 3 * num_deg, is_cos = gidx >= half, h = is_cos ? gidx - half : gidx;
    const float y = __fmul_rn(__ldg(vd + h % 3), __int_as_float((127 + h / 3) << 23));
    enc = sinf(is_cos ? __fadd_rn(y, MIPNERF_HALF_PI_F32) : y);
  }
  return enc;
}
__device__ __forceinline__ void level_view_terms(const LevelParams& p, int64_t tile, float* slot, int hw, int lane) {
  const float4* wt = reinterpret_cast<const float4*>(p.wimage + kViewDirOffset);  // [27][128] | bias[128]
  const float4 b4 = __ldg(wt + kViewDim * kCond / 4 + lane);
#pragma unroll 1
  for (int r = kViewPts * hw; r < kN; r += kViewPts * (kHelperThreads / 32)) {
    float enc[kViewPts];
#pragma unroll
    for (int q = 0; q < kViewPts; ++q) {
      const int64_t pt = tile * kN + r + q;
      enc[q] = 0.f;
      if (lane < kViewDim && pt < p.num_points) {
        const float* vd = p.viewdirs + pt * 3;
        if (lane < 3) {
          enc[q] = __ldg(vd + lane);  // append_identity
        } else {
          const int gidx = lane - 3, is_cos = gidx >= 12, h = is_cos ? gidx - 12 : gidx;  // scale-major, then xyz
          const float y = __fmul_rn(__ldg(vd + h % 3), __int_as_float((127 + h / 3) << 23));
          enc[q] = sinf(is_cos ? __fadd_rn(y, MIPNERF_HALF_PI_F32) : y);
        }
      }
    }
    float acc[kViewPts][4];
#pragma unroll
    for (int q = 0; q < kViewPts; ++q) acc[q][0] = b4.x, acc[q][1] = b4.y, acc[q][2] = b4.z, acc[q][3] = b4.w;
#pragma unroll 3
    for (int k = 0; k < kViewDim; ++k) {
      const float4 w4 = __ldg(wt + k * (kCond / 4) + lane);
#pragma unroll
      for (int q = 0; q < kViewPts; ++q) {
        const float e = __shfl_sync(0xffffffffu, enc[q], k);
        acc[q][0] = fmaf(w4.x, e, acc[q][0]);
        acc[q][1] = fmaf(w4.y, e, acc[q][1]);
        acc[q][2] = fmaf(w4.z, e, acc[q][2]);
        acc[q][3] = fmaf(w4.w, e, acc[q][3]);
      }
    }
#pragma unroll
    for (int q = 0; q < kViewPts; ++q)
      __stcg(reinterpret_cast<float4*>(slot + (r + q) * kCond) + lane,
             make_float4(acc[q][0], acc[q][1], acc[q][2], acc[q][3]));
  }
  __threadfence_block();
}

// ---- the helper warps' work (ht = helper thread 0..95, hw = helper warp 0..2) ----
// Tile tt of `ray` into the feature buffer fbuf: first (tt == 0) the ray prologue, once per ray, then the tile's
// features.  The prologue leaves the ray's view bias in its shared-memory slot vb_slot[128] for the consumers (computed
// at level 0, which also stores it to p.view_bias for the later levels; copied from p.view_bias otherwise, MLP-only
// mode included).  Its global stores (fenceposts, view bias) are read back by this CTA only, through L2 (ld.cg), by the
// helpers after the helper barrier.  Density-only mode: the tile's query points' features only.  Radiance mode: first
// the view-direction terms of the tile's points into its slot `vslot` (level_view_terms), then their features.
template <int kFmt, bool kX3, int kT, int kMode = kModeForward>
__device__ __forceinline__ void level_prepare_tile(const LevelParams& p, int64_t ray, int tt, uint8_t* fbuf,
                                                   float* rs_scratch, int ht, int hw, int lane, PhaseClock& clk,
                                                   float* vb_slot, float* vslot = nullptr) {
  constexpr int kNs = kT * kN;  // samples per ray
  constexpr bool kDensity = kMode != kModeForward;  // a query mode: the tile is 128 query points
  if constexpr (kMode == kModeRadiance) {
    level_view_terms(p, ray, vslot, hw, lane);
    clk.mark(kPhPrologue);
  }
  if (!kDensity && (kT == 1 || tt == 0)) {
    if (hw == 0) {
      float* t_ray = p.t + ray * (kNs + 1);
      if (p.t_mode == 1) {  // coarse fenceposts (bit-identical to coarse_t_kernel)
        const float nr = __ldg(p.near + ray), fr = __ldg(p.far + ray);
        const bool jit = draws_active(p.t_rand);
        for (int j = lane; j <= kNs; j += 32)
          __stcg(t_ray + j, coarse_fencepost(nr, fr, j, kNs, p.disparity, jit,
                                             jit ? draw_uniform(p.t_rand, ray, j, kNs + 1) : 0.f));
      } else if (p.t_mode == 2) {
        resample_warp_lean<true>(p.t_prev + ray * (kNs + 1), p.w_prev + ray * kNs, kNs, kNs + 1, p.randomized,
                                 p.u_jitter, ray, p.resample_padding, rs_scratch, t_ray,
                                 p.inds ? p.inds + ray * (kNs + 1) : nullptr, lane);
      }
    } else if (hw == 1 && p.vb_mode == 0) {  // the ray's view bias from p.view_bias into its slot
#pragma unroll
      for (int j = 0; j < 4; ++j) vb_slot[lane + 32 * j] = __ldcg(p.view_bias + ray * kCond + lane + 32 * j);
    } else if (hw == 1) {
      // per-ray view-layer bias  b[n] + W[n, 256:283] . pos_enc(viewdir)   (models/mip.py:353-363,
      // models/mip_nerf.py:106-108): lane f < 27 owns encoding element f, lane owns outputs n = lane + 32 j; into the
      // ray's slot, and into p.view_bias for the later levels
      float enc = 0.f;
      if (lane < kViewDim) {
        if (lane < 3) {
          enc = __ldg(p.viewdirs + ray * 3 + lane);  // append_identity
        } else {
          const int gidx = lane - 3, is_cos = gidx >= 12, h = is_cos ? gidx - 12 : gidx;  // scale-major, then xyz
          const float y = __fmul_rn(__ldg(p.viewdirs + ray * 3 + h % 3), __int_as_float((127 + h / 3) << 23));
          enc = sinf(is_cos ? __fadd_rn(y, MIPNERF_HALF_PI_F32) : y);
        }
      }
      const float* wt = reinterpret_cast<const float*>(p.wimage + kViewDirOffset);  // [27][128] | bias[128]
      float acc[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = __ldg(wt + kViewDim * kCond + lane + 32 * j);
#pragma unroll
      for (int k = 0; k < kViewDim; ++k) {
        const float e = __shfl_sync(0xffffffffu, enc, k);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = fmaf(__ldg(wt + k * kCond + lane + 32 * j), e, acc[j]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        vb_slot[lane + 32 * j] = acc[j];
        __stcg(p.view_bias + ray * kCond + lane + 32 * j, acc[j]);
      }
    }
    __threadfence_block();
    clk.mark(kPhPrologue);
    if (p.t_mode != 0 || p.vb_mode != 0) {  // the prologue's global stores are read back after the helper barrier
      named_bar_sync(kHelperBar, kHelperThreads);
      clk.mark(kPhBarrier);
    }
  }
  // Gaussians + IPE features: 128 rows x 3 parts of two 8-feature groups = 384 units, four per helper thread; a warp's
  // 32 units share their part
  RayGeom g{};
  if (!kDensity && !p.feat_in) g = load_ray_geom(p.origins, p.directions, p.radii, ray);
  const int row0 = kT == 1 ? 0 : tt * kN;  // the tile's first row of the ray
#pragma unroll 1
  for (int u = ht; u < 3 * kN; u += kHelperThreads) {
    const int row = u & (kN - 1), part = u / kN;
    float t0 = 0.f, t1 = 0.f;
    if (!kDensity && !p.feat_in)
      t0 = __ldcg(p.t + ray * (kNs + 1) + row0 + row), t1 = __ldcg(p.t + ray * (kNs + 1) + row0 + row + 1);
    ipe_row_group<kFmt, kX3, kT, kDensity>(p, g, ray, row, t0, t1, fbuf, 2 * part, 2 * part + 2);
  }
  fence_proxy_async_smem();  // the features are read by wgmma (async proxy)
  clk.mark(kPhIpe);
}

// Activations + compositing of `ray` from its raw heads hd[128 kT][4] (or, in MLP-only mode, the raw heads out), with
// the summation order of a thread-per-row warpgroup: rows in 4 kT chunks of 32, chunk q on helper warp q % 3, each
// chunk scanned / reduced within its warp, the chunks' carries and partial sums added in chunk order, across the tile
// boundary too.  One round per tile (chunks 4 u .. 4 u + 3 of tile u); each helper thread arrives on heads_empty[u]
// once it has read its rows of tile u's heads.
template <int kT>
__device__ __forceinline__ void level_composite_ray(const LevelParams& p, int64_t ray, const float* hd,
                                                    uint64_t* heads_empty, float* cs, float* ps, int ht, int hw,
                                                    int lane, PhaseClock& clk) {
  constexpr int kNs = kT * kN;  // samples per ray
  if (kT == 1 && p.raw_rgb_out) {  // MLP-only mode: hand back the raw heads (models/mip_nerf.py:98,110)
    for (int row = ht; row < kN; row += kHelperThreads) {
      const float4 h4 = *reinterpret_cast<const float4*>(hd + row * 4);
      const int64_t sidx = ray * kN + row;
      p.raw_rgb_out[sidx * 3 + 0] = h4.y + c_small.b_color[0];
      p.raw_rgb_out[sidx * 3 + 1] = h4.z + c_small.b_color[1];
      p.raw_rgb_out[sidx * 3 + 2] = h4.w + c_small.b_color[2];
      p.raw_density_out[sidx] = h4.x + c_small.b_density;
    }
    mbar_arrive(heads_empty);
    clk.mark(kPhComposite);
    return;
  }
  const float* t_ray = p.t + ray * (kNs + 1);
  const float dx = __ldg(p.directions + ray * 3), dy = __ldg(p.directions + ray * 3 + 1),
              dz = __ldg(p.directions + ray * 3 + 2);
  const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
  constexpr int kChunksPerWarp = 2;  // chunks hw, hw + 3 of a tile
#pragma unroll 1
  for (int u = 0; u < kT; ++u) {
    float dd[kChunksPerWarp], excl[kChunksPerWarp], crgb[kChunksPerWarp][3], tmid[kChunksPerWarp];
#pragma unroll
    for (int k = 0; k < kChunksPerWarp; ++k) {
      const int q = hw + 3 * k, row = 32 * (4 * u + q) + lane;  // row of the ray
      if (q >= 4) break;
      const float4 h4 = *reinterpret_cast<const float4*>(hd + row * 4);
      const int64_t sidx = ray * kNs + row;
      float raw_dens = h4.x + c_small.b_density;
      if (draws_active(p.dnoise))  // models/mip_nerf.py:232-233
        raw_dens = noisy_raw_density<kNs>(raw_dens, p.dnoise, ray, row);
      if (kT == 1 && p.raw_rgb_keep) {  // training: the raw heads as well (render_backward recomputes the rest; the
        p.raw_rgb_keep[sidx * 3 + 0] = h4.y + c_small.b_color[0];  // density head WITH its noise, so that softplus'
        p.raw_rgb_keep[sidx * 3 + 1] = h4.z + c_small.b_color[1];  // is taken at the same point)
        p.raw_rgb_keep[sidx * 3 + 2] = h4.w + c_small.b_color[2];
        p.raw_density_keep[sidx] = raw_dens;
      }
      const float t0 = __ldcg(t_ray + row), t1 = __ldcg(t_ray + row + 1);
      const float density = density_activation(raw_dens, p.density_bias);
      crgb[k][0] = rgb_activation(h4.y + c_small.b_color[0], p.rgb_scale, p.rgb_padding);
      crgb[k][1] = rgb_activation(h4.z + c_small.b_color[1], p.rgb_scale, p.rgb_padding);
      crgb[k][2] = rgb_activation(h4.w + c_small.b_color[2], p.rgb_scale, p.rgb_padding);
      tmid[k] = 0.5f * (t0 + t1);
      dd[k] = density * ((t1 - t0) * dnorm);
      float incl = dd[k];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
      }
      excl[k] = __shfl_up_sync(0xffffffffu, incl, 1);
      if (lane == 0) excl[k] = 0.f;
      if (lane == 31) cs[4 * u + q] = incl;
    }
    mbar_arrive(heads_empty + u);
    clk.mark(kPhComposite);
    named_bar_sync(kHelperBar, kHelperThreads);
    clk.mark(kPhBarrier);
#pragma unroll
    for (int k = 0; k < kChunksPerWarp; ++k) {
      const int q = hw + 3 * k, qr = 4 * u + q;  // chunk of the tile, of the ray
      if (q >= 4) break;
      float before = 0.f;
      for (int qq = 0; qq < qr; ++qq) before += cs[qq];
      const float w = -expm1f(-dd[k]) * expf(-(before + excl[k]));
      p.weights[ray * kNs + 32 * qr + lane] = w;
      const float pr = warp_sum(w * crgb[k][0]), pg = warp_sum(w * crgb[k][1]), pb = warp_sum(w * crgb[k][2]),
                  pw = warp_sum(w), pd = warp_sum(w * tmid[k]);
      if (lane == 0) {
        float* dst = ps + qr * 8;
        dst[0] = pr, dst[1] = pg, dst[2] = pb, dst[3] = pw, dst[4] = pd;
      }
    }
  }
  clk.mark(kPhComposite);
  named_bar_sync(kHelperBar, kHelperThreads);
  clk.mark(kPhBarrier);
  if (ht == 0) {
    float s[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    for (int qq = 0; qq < 4 * kT; ++qq)
      for (int k = 0; k < 5; ++k) s[k] += ps[qq * 8 + k];
    const float t_first = __ldcg(t_ray), t_last = __ldcg(t_ray + kNs);
    float d = s[4];
    if (isnan(d)) d = 0.f;
    else if (isinf(d)) d = d > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
    d = fminf(fmaxf(d, t_first), t_last);
    const float bg = p.white_bkgd ? 1.0f - s[3] : 0.f;
    p.comp_rgb[ray * 3 + 0] = s[0] + bg;
    p.comp_rgb[ray * 3 + 1] = s[1] + bg;
    p.comp_rgb[ray * 3 + 2] = s[2] + bg;
    p.distance[ray] = d;
    p.acc[ray] = s[3];
  }
  clk.mark(kPhComposite);
  named_bar_sync(kHelperBar, kHelperThreads);  // ht 0 has consumed ps / everyone cs before the next ray reuses them
  clk.mark(kPhBarrier);
}

// Density-only mode: the raw density of tile `tile`'s query points from its raw heads hd[128][4] (the sum MLP-only mode
// hands back, models/mip_nerf.py:98) and its activation (models/mip_nerf.py:237); rows past the last point are masked.
__device__ __forceinline__ void level_density_out(const LevelParams& p, int64_t tile, const float* hd,
                                                  uint64_t* heads_empty, int ht, PhaseClock& clk) {
  for (int row = ht; row < kN; row += kHelperThreads) {
    const int64_t pt = tile * kN + row;
    if (pt >= p.num_points) break;
    const float raw = hd[row * 4] + c_small.b_density;
    if (p.raw_density_out) p.raw_density_out[pt] = raw;
    if (p.density_out) p.density_out[pt] = density_activation(raw, p.density_bias);
  }
  mbar_arrive(heads_empty);
  clk.mark(kPhComposite);
}

// Radiance mode: tile `tile`'s raw heads hd[128][4] plus the head biases (the sums MLP-only mode hands back,
// models/mip_nerf.py:98,110) and their activations (models/mip_nerf.py:236-237); rows past the last point are masked.
__device__ __forceinline__ void level_radiance_out(const LevelParams& p, int64_t tile, const float* hd,
                                                   uint64_t* heads_empty, int ht, PhaseClock& clk) {
  for (int row = ht; row < kN; row += kHelperThreads) {
    const int64_t pt = tile * kN + row;
    if (pt >= p.num_points) break;
    const float4 h4 = *reinterpret_cast<const float4*>(hd + row * 4);
    const float raw[4] = {h4.x + c_small.b_density, h4.y + c_small.b_color[0], h4.z + c_small.b_color[1],
                          h4.w + c_small.b_color[2]};
    if (p.raw_density_out) p.raw_density_out[pt] = raw[0];
    if (p.density_out) p.density_out[pt] = density_activation(raw[0], p.density_bias);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      if (p.raw_rgb_out) p.raw_rgb_out[pt * 3 + ch] = raw[1 + ch];
      if (p.rgb_out) p.rgb_out[pt * 3 + ch] = rgb_activation(raw[1 + ch], p.rgb_scale, p.rgb_padding);
    }
  }
  mbar_arrive(heads_empty);
  clk.mark(kPhComposite);
}

// kMode = kModeDensity (kT = 1): density-only mode.  The producer streams the stages of layers 0-7 only (a prefix of
// the image), the consumers run layers 0-7 and finish the density head in layer 7's epilogue, and the helpers encode
// the query points and write the densities; everything else is the forward's schedule.
// kMode = kModeRadiance (kT = 1): radiance mode.  The producer and the consumers run the forward's schedule, except that
// the view layer's epilogue adds to each row its own point's view-direction term instead of one per-ray bias.  The
// helpers write those terms (level_view_terms) and the features of tile i ahead of the consumers, and the raw heads and
// activations of tile i - 1 after them.  The terms of tile i go to slot i % 2 of this CTA; two slots are enough: the
// helpers write slot i % 2 for tile i only after they have waited on heads_full of tile i - 2 (in the previous round
// of their loop, with one feature buffer or two), and the consumers arrive on heads_full of a tile only after its view
// layer's epilogue has read the tile's terms (the quad sums that the arriving thread stores depend on every loaded term).
// kMode = kModeViewAcc (kT = 1): view-accumulator mode.  The producer and the consumers run radiance mode's schedule
// through the view layer's K-slabs (the same stages and wgmmas into acc0, in the same order), then the consumers store
// acc0 as it is to p.view_acc instead of the view-layer epilogue and the colour head; the density head is finished and
// handed over as in radiance mode.  The helpers compute no view terms: they encode the query points and write the
// densities, as in density-only mode.
// kMode = kModeForward: the per-ray view bias of the i-th ray of the CTA is in shared-memory slot vbias[i % 2], which
// the helpers fill in the ray prologue of its tile 0 and the view-layer epilogues of all its tiles read.  The same
// argument holds per ray: the helpers fill the slot of ray i only after they have waited on heads_full of every tile of
// ray i - 2 (in round i - 1 of their loop, with kT = 1 or 2 and one feature buffer or two), and the consumers arrive on
// heads_full of a tile only after its view-layer epilogue has read the slot; the slot of ray i is written before the
// feat_full arrive of its tile 0, which the consumers wait on before any tile of ray i.
// kTrain (bf16x3 / fp16x3 forward with the training dump only): the dump also carries the lo halves of the split
// activation tiles, at act_dump + 9 dump_tiles 64 KB (same [9][dump_tiles] layout), and of the view-layer output, at
// v_dump + dump_tiles 32 KB.  A compile-time flag, so that the inference instantiations carry none of it.
// kQueryDump (bf16 / fp16 query modes, the backward of a query only): the query tiles leave the training forward's dump,
// tile = query tile of the launch: h_0..h_7 (density mode: h_7 from layer 7's epilogue, which otherwise only finishes
// the density head) and, in radiance mode, the bottleneck into act_dump, the view-layer output into v_dump.  The raw
// heads are the query's own outputs.  Rows past the last point hold the features of a zero Gaussian: finite.
template <int kFmt, bool kX3, int kT, int kMode = kModeForward, bool kTrain = false, bool kQueryDump = false>
__global__ void __launch_bounds__(kThreads, 1) mlp_level_kernel(const LevelParams p) {
  static_assert(!kTrain || (kX3 && kT == 1 && kMode == kModeForward), "the split training forward: 128 samples");
  static_assert(!kQueryDump || (!kX3 && kT == 1 && kMode != kModeForward), "the 16-bit query modes' dump");
  constexpr bool kDensity = kMode == kModeDensity;
  constexpr bool kQuery = kMode != kModeForward;  // density or radiance: 128 query points per tile
  constexpr bool kDumps = !kQuery || kQueryDump;  // the training dump (p.act_dump, p.v_dump) may be set
  static_assert(!kQuery || kT == 1, "the query modes take one 128-point tile at a time");
  using Lay = LevelLayout<kX3, kT>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* sA = smem + Lay::kA;
  uint8_t* sF = smem + Lay::kF;
  uint8_t* sW = smem + Lay::kW;
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + Lay::kMisc);  // [kStages] producer -> consumers (tx bytes)
  uint64_t* w_empty = w_full + Lay::kStages;                           // [kStages] consumers (2 arrives) -> producer
  uint64_t* feat_full = w_empty + Lay::kStages;     // [kFeatBufs] helpers (kHelperThreads arrives) -> consumers
  uint64_t* feat_empty = feat_full + Lay::kFeatBufs;  // [kFeatBufs] consumers (2 arrives) -> helpers
  uint64_t* heads_full = feat_empty + Lay::kFeatBufs;  // [2] consumers (kHeadsWriters arrives) -> helpers
  uint64_t* heads_empty = heads_full + 2;              // [2] helpers (kHelperThreads arrives) -> consumers
  float* heads = reinterpret_cast<float*>(heads_empty + 2);  // [2][128][4] raw density, rgb dots
  float* cs = heads + 2 * kN * 4;                            // [4 kT] scan carries
  float* ps = cs + 4 * kT;                                   // [4 kT][8] partial sums
  float* rs_scratch = ps + 32 * kT;                          // [128 kT + 1] resampler scratch
  float* vbias = reinterpret_cast<float*>(smem + Lay::kVBias);  // [2][128] forward: per-ray view bias (ray parity)
  unsigned long long* phase_rows = reinterpret_cast<unsigned long long*>(smem + Lay::kPhase);
  const int phase_slot = p.t_mode == 2 ? 1 : 0;
  PhaseClock clk;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < Lay::kStages; ++i) {
      mbar_init(&w_full[i], 1);
      mbar_init(&w_empty[i], 2);
    }
    for (int i = 0; i < Lay::kFeatBufs; ++i) {
      mbar_init(&feat_full[i], kHelperThreads);
      mbar_init(&feat_empty[i], 2);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&heads_full[i], kHeadsWriters);
      mbar_init(&heads_empty[i], kHelperThreads);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(kProducerRegs) : "memory");
    if (warp >= kHelperWarp0) {
      // ============================ helpers (warps 9-11): a two-stage ray pipeline ============================
      // prepare tile 0 of ray i (into feature buffer j % kFeatBufs, j the tile's index in the CTA, once the consumers
      // are done with its previous tile), composite ray i - 1, then prepare the other tile of ray i; the consumers
      // meanwhile run the layers of the tiles of ray i - 1 and then of ray i.  With kT = 2 the raw heads of a ray's
      // tiles 0 / 1 are in heads[0] / heads[1], i.e. rows 0..255 of heads.
      const int ht = tid - 32 * kHelperWarp0, hw = warp - kHelperWarp0;
      clk.begin(phase_rows + 3 * kNumPhases, ht == 0);
      for (int64_t ray = blockIdx.x, i = 0;; ray += gridDim.x, ++i) {
        const bool more = ray < p.num_rays;
#pragma unroll 1
        for (int tt = 0; tt < kT; ++tt) {
          const int64_t j = i * kT + tt;
          if (more) {
            const int fb = (int)(j % Lay::kFeatBufs);
            mbar_wait(&feat_empty[fb], ((uint32_t)(j / Lay::kFeatBufs) & 1u) ^ 1u);
            clk.mark(kPhFeatEmpty);
            level_prepare_tile<kFmt, kX3, kT, kMode>(
                p, ray, tt, sF + fb * Lay::kFBuf, rs_scratch, ht, hw, lane, clk, vbias + (i & 1) * kCond,
                kMode == kModeRadiance ? p.view_bias + ((size_t)blockIdx.x * 2 + (j & 1)) * (kN * kCond) : nullptr);
            mbar_arrive(&feat_full[fb]);
          }
          if (tt == 0 && i > 0) {  // ray - gridDim.x, the (i - 1)-th ray of the CTA: tiles (i - 1) kT ..
            const int par = (int)(((i - 1) * kT) & 1);  // kT = 2: 0
#pragma unroll
            for (int u = 0; u < kT; ++u)
              mbar_wait(&heads_full[par + u], (uint32_t)(((i - 1) * kT + u) >> 1) & 1u);
            clk.mark(kPhHeadsFull);
            if constexpr (kDensity || kMode == kModeViewAcc)
              level_density_out(p, ray - gridDim.x, heads + par * kN * 4, &heads_empty[par], ht, clk);
            else if constexpr (kMode == kModeRadiance)
              level_radiance_out(p, ray - gridDim.x, heads + par * kN * 4, &heads_empty[par], ht, clk);
            else
              level_composite_ray<kT>(p, ray - gridDim.x, heads + par * kN * 4, &heads_empty[par], cs, ps, ht, hw, lane,
                                      clk);
          }
        }
        if (!more) break;
      }
      clk.end(phase_slot, 3);
      return;
    }
    // ============================ weight producer (warp 8, one lane) ============================
    if (lane == 0) {
      clk.begin(phase_rows + 2 * kNumPhases, true);
      int st = 0;
      uint32_t ph = 0;
      const uint64_t pol = l2_policy_evict_last();  // the image is re-read by every CTA for every ray
      for (int64_t tile = 0, ray = blockIdx.x; ray < p.num_rays; ray += ++tile % kT == 0 ? gridDim.x : 0) {
        const uint8_t* src = p.wimage;  // the stages are contiguous in issue order (w_stages_contiguous)
        for (int l = 0; l < (kDensity ? 8 : kNumLayers); ++l)
          for (int h = 0; h < num_halves(l); ++h)  // N-half major, then K-slab
            for (int s = 0; s < num_slabs(!kX3, l); ++s) {
              const uint32_t bytes = w_stage(!kX3, l, s).bytes;
              clk.mark(kPhIssue);
              mbar_wait(&w_empty[st], ph ^ 1);
              clk.mark(kPhWEmpty);
              mbar_arrive_expect_tx(&w_full[st], kX3 ? 2 * bytes : bytes);
              bulk_g2s_hint(sW + st * Lay::kStage, src, bytes, &w_full[st], pol);
              if (kX3) bulk_g2s_hint(sW + st * Lay::kStage + bytes, src + kLoOffset, bytes, &w_full[st], pol);
              src += bytes;
              if (++st == Lay::kStages) {
                st = 0;
                ph ^= 1;
              }
            }
      }
      clk.mark(kPhIssue);
      clk.end(phase_slot, 2);
    }
    return;
  }

  // ============================ consumer warpgroups ============================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(kConsumerRegs) : "memory");
  const int wg = warp >> 2, t = tid & 127, wq = warp & 3;
  const int r0 = 64 * wg + 16 * wq + (lane >> 2);  // accumulator rows r0, r0 + 8 of this thread
  const int cq = 2 * (lane & 3);                   // and columns 8 j + cq, + 1
  const bool leader = t == 0;
  const SmallParams* __restrict__ gsp = reinterpret_cast<const SmallParams*>(p.wimage + kSmallOffset);
  const uint32_t a_u = smem_u32(sA) + (uint32_t)wg * 64u * 128u;
  const uint32_t w_u = smem_u32(sW);
  // the training forward's dump (p.act_dump, p.v_dump) exists for kT = 1 only
  const uint64_t dump_policy =
      (kMode != kModeRadiance || kQueryDump) && kT == 1 && p.act_dump ? l2_policy_evict_first() : 0ull;  // must not evict the weights
  bool dump_pending = false;
  RingPos rp{0, 0u, -1};
  clk.begin(phase_rows + wg * kNumPhases, leader);
  // tile i of the CTA is tile i % kT of `ray`; every tile of a ray adds the ray's one view bias
  for (int64_t ray = blockIdx.x, i = 0; ray < p.num_rays; ray += ++i % kT == 0 ? gridDim.x : 0) {
    // the tile's feature buffer and raw-heads parity, and their mbarrier phases
    const int fb = (int)(i % Lay::kFeatBufs), par = (int)(i & 1);
    const uint32_t fph = (uint32_t)(i / Lay::kFeatBufs) & 1u, hph = (uint32_t)(i >> 1) & 1u;
    const int vpar = kT == 1 ? par : (int)hph;  // the ray's view-bias slot: the parity of i / kT
    // this warpgroup's rows of the tile's feature buffer (SW128 slab, SW64 tail)
    const uint32_t f_u = smem_u32(sF) + (uint32_t)fb * Lay::kFBuf + (uint32_t)wg * 64u * 128u;
    const uint32_t ft_u = smem_u32(sF) + (uint32_t)fb * Lay::kFBuf + kStageBytes + (uint32_t)wg * 64u * 64u;
    mbar_wait(&feat_full[fb], fph);
    clk.mark(kPhFeatFull);

    float d0 = 0.f, d1 = 0.f;  // density head, rows r0 / r0 + 8 (partial over this thread's columns)
    float rgb[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    // ---- the layers, software-pipelined so that each epilogue runs under wgmmas instead of after them.  In the split
    // modes the epilogue of trunk layer / bottleneck l overwrites, in place, the activation columns (hi and lo tiles)
    // that layer l read; wgmmas consume K in order, and K-slab s of layers 1..9 reads only columns 32 s .. 32 s + 31
    // (layer 5's slabs 8-10 and layer 0 read the feature tile).  Per layer l:
    //   1. N-half 0 into acc0: K-slabs 0..3 were issued under the previous layer's acc1 epilogue (step 4); the rest here.
    //   2. N-half 1 into acc1; after K-slab kEpiOverlap + c has been committed and waited for, chunk c of acc0's
    //      epilogue (columns 32 c .. 32 c + 31).  That wait leaves only K-slab kEpiOverlap + c in flight: all of N-half
    //      0 has retired (acc0 is final), and so has K-slab c of N-half 1, the last reader of those columns.  Layer 0
    //      reads none of the columns it writes, so its chunks follow K-slabs 0, 1, 2, 2.
    //   3. fence + barrier: columns 0..127 of layer l + 1's input are complete for this warpgroup's rows.
    //   4. Layer l + 1's N-half 0, K-slabs 0..3 (columns 0..127 only); the chunks of acc1's epilogue (columns 128..255)
    //      follow the waits of K-slabs 0, 1, 2, 2, and K-slab 3 runs under the barrier instead of a chunk.  The first
    //      wait retires all of layer l.
    //   5. fence + barrier: layer l + 1's input is complete (and goes out with bulk stores in the training forward).
    // A chunk's bias loads are issued before the K-slab it follows.  The wgmmas into each accumulator, their operands and
    // order, and the epilogue arithmetic are those of an unpipelined loop, so the results are the same bit for bit.
    // bf16 / fp16 keep the layer input in registers instead (below): the same steps without 3 and 5.
    float acc0[64], acc1[64];
    wgmma_fence_acc(acc0);
#pragma unroll
    for (int s = 0; s < num_slabs(!kX3, 0); ++s)
      level_mma_slab<kFmt, kX3>(acc0, 0, s, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
    if constexpr (!kX3) {
      // bf16 / fp16: the layers are chained through registers (wgmma with A from registers), the schedule above with
      // no activation tile and 64-wide K-slabs: each epilogue chunk writes its 16-bit pairs into the A fragments of the
      // next layer's input, one of two arrays (layer l reads xa or xb, writes the other), so no layer's writes touch
      // what its own wgmmas read, and there is no fence or barrier between layers.  acc0's chunks follow N-half 1's
      // K-slabs epi_slab_acc0(c) and acc1's the next layer's K-slabs 0, 1.  Layer 0 and layer 5's K-slabs 4, 5 read the
      // feature tile; layer 0 has two K-slabs (64 wide + the 32-wide tail), and two of its acc0 chunks follow each.  The
      // training forward's activation tiles go out from the epilogue's registers.
      const LevelRsCtx k{f_u, ft_u, w_u, w_full, w_empty, &feat_empty[fb], gsp,
                         kDumps && kT == 1 && p.act_dump ? p.act_dump + (size_t)ray * kABytes : nullptr,
                         (size_t)p.dump_tiles * kABytes, dump_policy, r0, cq, leader};
      uint32_t xa[64], xb[64];
      static_assert(2 * num_slabs(true, 0) == kEpiChunks, "layer 0: two acc0 chunks after each of its K-slabs");
      wgmma_fence_acc(acc1);
#pragma unroll
      for (int s = 0; s < num_slabs(true, 0); ++s) {
        EpiConsts e[2];
        level_epilogue_consts(e[0], 0, 0, 2 * s, cq, gsp);
        level_epilogue_consts(e[1], 0, 0, 2 * s + 1, cq, gsp);
        level_mma_slab<kFmt, false>(acc1, 0, s, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
        if (s == 0) wgmma_fence_acc(acc0);
        level_epilogue_chunk_rs<kFmt>(acc0, e[0], 0, 0, 2 * s, xb, k, d0, d1);
        level_epilogue_chunk_rs<kFmt>(acc0, e[1], 0, 0, 2 * s + 1, xb, k, d0, d1);
        clk.mark(kPhEpilogue);
      }
      level_rs_next_head<kFmt>(acc0, acc1, xb, 0, false, k, rp, clk, d0, d1);
#pragma unroll 1
      for (int l = 1; l < (kDensity ? 7 : 9); l += 2) {
        level_rs_layer<kFmt, true>(acc0, acc1, xb, xa, l, k, rp, clk, d0, d1);
        level_rs_layer<kFmt, false>(acc0, acc1, xa, xb, l + 1, k, rp, clk, d0, d1);
      }
      if constexpr (kDensity) {
        level_rs_layer<kFmt, false, true>(acc0, acc1, xb, xa, 7, k, rp, clk, d0, d1);
      } else {
        // the rest of the view layer's one N-half, from the bottleneck in xb
#pragma unroll
        for (int s = 2; s < num_slabs(true, 9); ++s)
          level_mma_slab_rs<kFmt>(acc0, xb, s, w_u, w_full, w_empty, rp, leader, clk);
      }
    } else {
      for (int l = 0; l < 9; ++l) {
        // 1. the rest of N-half 0
        if (l > 0)
          for (int s = kEpiChunks; s < num_slabs(false, l); ++s)
            level_mma_slab<kFmt, kX3>(acc0, l, s, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
        // 2. N-half 1, with acc0's epilogue under it
        wgmma_fence_acc(acc1);
        const int first = l == 0 ? 0 : kEpiOverlap;  // K-slab that carries chunk 0
        for (int s = 0; s < first; ++s)
          level_mma_slab<kFmt, kX3>(acc1, l, s, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
#pragma unroll
        for (int c = 0; c < kEpiChunks; ++c) {
          EpiConsts e;
          level_epilogue_consts(e, l, 0, c, cq, gsp);
          if (first + c < num_slabs(false, l))
            level_mma_slab<kFmt, kX3>(acc1, l, first + c, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
          if (c == 0) {
            wgmma_fence_acc(acc0);
            if (dump_pending) {  // the previous tile's bulk stores must have READ it before it is overwritten
              if (leader) bulk_store_wait_read();
              dump_pending = false;
              clk.mark(kPhEpilogue);
              named_bar_sync(1 + wg, 128);
              clk.mark(kPhBarrier);
            }
          }
          level_epilogue_chunk<kFmt, kX3>(acc0, e, l, 0, c, r0, cq, sA, gsp, d0, d1);
          clk.mark(kPhEpilogue);
        }
        for (int s = first + kEpiChunks; s < num_slabs(false, l); ++s)
          level_mma_slab<kFmt, kX3>(acc1, l, s, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
        if (kDensity && l == 7) break;  // density-only mode: layer 7 has no next layer (acc1's epilogue below)
        // 3.
        fence_proxy_async_smem();
        clk.mark(kPhEpilogue);
        named_bar_sync(1 + wg, 128);
        clk.mark(kPhBarrier);
        // 4. the next layer's N-half 0, K-slabs 0..3, with acc1's epilogue under the first three
        wgmma_fence_acc(acc0);
#pragma unroll
        for (int c = 0; c < kEpiChunks; ++c) {
          EpiConsts e;
          level_epilogue_consts(e, l, 128, c, cq, gsp);
          if (c < kEpiChunks - 1) {
            level_mma_slab<kFmt, kX3>(acc0, l + 1, c, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
            if (c == 0 && l == 5 && leader) mbar_arrive(&feat_empty[fb]);  // layer 5's skip slabs have retired
            if (c == 0) wgmma_fence_acc(acc1);
          }
          level_epilogue_chunk<kFmt, kX3>(acc1, e, l, 128, c, r0, cq, sA, gsp, d0, d1);
          clk.mark(kPhEpilogue);
        }
        level_mma_slab<kFmt, kX3>(acc0, l + 1, kEpiChunks - 1, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
        // 5.
        fence_proxy_async_smem();
        clk.mark(kPhEpilogue);
        named_bar_sync(1 + wg, 128);
        clk.mark(kPhBarrier);
        if (kMode != kModeRadiance && kT == 1 && p.act_dump) {  // training forward: this warpgroup's rows of the 16-bit tile, as the tensor core
          // reads it
          if (leader) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint32_t o = (uint32_t)k * kStageBytes + (uint32_t)wg * 8192u;
              bulk_s2g_hint(p.act_dump + ((size_t)l * p.dump_tiles + ray) * kABytes + o, sA + o, 8192u, dump_policy);
              if constexpr (kTrain)
                bulk_s2g_hint(p.act_dump + ((size_t)(9 + l) * p.dump_tiles + ray) * kABytes + o, sA + kABytes + o, 8192u,
                              dump_policy);
            }
          }
          dump_pending = true;
          clk.mark(kPhEpilogue);
        }
      }
      if constexpr (kDensity) {  // layer 7's acc1 epilogue, as step 4 runs it
        wgmma_wait<0>();
        wgmma_fence_acc(acc1);
        if (leader) mbar_arrive(&w_empty[rp.prev]);
        rp.prev = -1;
        clk.mark(kPhMma);
#pragma unroll
        for (int c = 0; c < kEpiChunks; ++c) {
          EpiConsts e;
          level_epilogue_consts(e, 7, 128, c, cq, gsp);
          level_epilogue_chunk<kFmt, kX3>(acc1, e, 7, 128, c, r0, cq, sA, gsp, d0, d1);
        }
        clk.mark(kPhEpilogue);
      } else {
        // the rest of the view layer's one N-half
        for (int s = kEpiChunks; s < num_slabs(false, 9); ++s)
          level_mma_slab<kFmt, kX3>(acc0, 9, s, a_u, f_u, ft_u, w_u, w_full, w_empty, rp, leader, clk);
      }
    }
    if constexpr (kMode == kModeViewAcc) {
      // the view layer's accumulators as they are, straight from the registers (evict-first: read once, by the pair
      // kernel, after this launch)
      wgmma_wait<0>();
      wgmma_fence_acc(acc0);
      if (leader) mbar_arrive(&w_empty[rp.prev]);
      rp.prev = -1;
      clk.mark(kPhMma);
      const uint64_t pol = l2_policy_evict_first();
      float* va = p.view_acc + ((size_t)ray * kN + r0) * kCond + cq;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        st_global_v2_hint(va + 8 * j, acc0[4 * j], acc0[4 * j + 1], pol);
        st_global_v2_hint(va + 8 * kCond + 8 * j, acc0[4 * j + 2], acc0[4 * j + 3], pol);
      }
    } else if constexpr (!kDensity) {
      // the view layer's epilogue from the registers; the forward reads its columns of the ray's view bias from the
      // ray's slot, in bf16 / fp16 while the last K-slab's wgmmas run (the split modes' training forward has no
      // registers to spare there: ptxas spills 32 values)
      const float* vs = vbias + vpar * kCond + cq;
      float2 vbr[16];
      if constexpr (kMode == kModeForward && !kX3) {
#pragma unroll
        for (int j = 0; j < 16; ++j) vbr[j] = *reinterpret_cast<const float2*>(vs + 8 * j);
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc0);
      if (leader) mbar_arrive(&w_empty[rp.prev]);
      rp.prev = -1;
      clk.mark(kPhMma);
      // view layer + colour head (models/mip_nerf.py:106-110); view bias = the per-ray view-direction term (radiance
      // mode: row r0 of the tile's global slot; row r0 + 8 adds its own term b1)
      const float* vb = p.view_bias + ((size_t)blockIdx.x * 2 + par) * (kN * kCond) + (size_t)r0 * kCond;
      uint8_t* vd = kDumps && kT == 1 && p.v_dump ? p.v_dump + (size_t)ray * (2 * kStageBytes) : nullptr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = 8 * j + cq;
        const float2 b = kMode == kModeRadiance ? __ldcg(reinterpret_cast<const float2*>(vb + c))
                         : kX3                  ? *reinterpret_cast<const float2*>(vs + 8 * j)
                                                : vbr[j];
        const float2 b1 = kMode == kModeRadiance ? __ldcg(reinterpret_cast<const float2*>(vb + 8 * kCond + c)) : b;
        float y[4] = {acc0[4 * j], acc0[4 * j + 1], acc0[4 * j + 2], acc0[4 * j + 3]};
        fadd2(y[0], y[1], b.x, b.y);
        fadd2(y[2], y[3], b1.x, b1.y);
#pragma unroll
        for (int e = 0; e < 4; ++e) y[e] = fmaxf(y[e], 0.f);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          const float2 wc = __ldg(reinterpret_cast<const float2*>(gsp->w_color[ch] + c));
          ffma2(rgb[0][ch], rgb[1][ch], y[0], y[2], wc.x, wc.x);
          ffma2(rgb[0][ch], rgb[1][ch], y[1], y[3], wc.y, wc.y);
        }
        if (vd) {  // training: the 16-bit view-layer output, same tile layout as the trunk's activation slabs
          *reinterpret_cast<uint32_t*>(vd + (c >> 6) * kStageBytes + sw128_offset(r0, c & 63)) = pack2<kFmt>(y[0], y[1]);
          *reinterpret_cast<uint32_t*>(vd + (c >> 6) * kStageBytes + sw128_offset(r0 + 8, c & 63)) =
              pack2<kFmt>(y[2], y[3]);
          if constexpr (kTrain) {  // and its lo halves
            uint8_t* vl = vd + (size_t)p.dump_tiles * (2 * kStageBytes);
            *reinterpret_cast<uint32_t*>(vl + (c >> 6) * kStageBytes + sw128_offset(r0, c & 63)) =
                pack2_low<kFmt>(y[0], y[1], pack2<kFmt>(y[0], y[1]));
            *reinterpret_cast<uint32_t*>(vl + (c >> 6) * kStageBytes + sw128_offset(r0 + 8, c & 63)) =
                pack2_low<kFmt>(y[2], y[3], pack2<kFmt>(y[2], y[3]));
          }
        }
      }
    }
    // ---- raw heads of this thread's two rows -> shared memory
    d0 = quad_sum(d0), d1 = quad_sum(d1);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) rgb[0][ch] = quad_sum(rgb[0][ch]), rgb[1][ch] = quad_sum(rgb[1][ch]);
    // one thread per quad: wait until the helpers have composited the ray two back, store, hand the rows over
    if ((lane & 3) == 0) {
      float* hd = heads + par * kN * 4;
      clk.mark(kPhEpilogue);
      mbar_wait(&heads_empty[par], hph ^ 1);
      clk.mark(kPhBarrier);
      *reinterpret_cast<float4*>(hd + r0 * 4) = make_float4(d0, rgb[0][0], rgb[0][1], rgb[0][2]);
      *reinterpret_cast<float4*>(hd + (r0 + 8) * 4) = make_float4(d1, rgb[1][0], rgb[1][1], rgb[1][2]);
      mbar_arrive(&heads_full[par]);
    }
    clk.mark(kPhEpilogue);
  }
  if (dump_pending && leader) bulk_store_wait_all();  // the last tile's store has left shared memory
  clk.mark(kPhEpilogue);
  clk.end(phase_slot, wg);
}

// MLP-only mode: same per-ray bias from a caller-supplied [B,27] view encoding
__global__ void view_bias_from_enc_kernel(const float* __restrict__ venc, const float* __restrict__ w,
                                          const float* __restrict__ b, float* __restrict__ out, int64_t num_rays) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= num_rays * kCond) return;
  const int64_t ray = idx / kCond;
  const int n = (int)(idx % kCond);
  float acc = __ldg(b + n);
#pragma unroll
  for (int k = 0; k < kViewDim; ++k)
    acc = fmaf(__ldg(w + (size_t)n * (kWidth + kViewDim) + kWidth + k), __ldg(venc + ray * kViewDim + k), acc);
  out[idx] = acc;
}

// Radiance under a shared direction set: the view-direction term  b_view[n] + sum_k W(k, n) enc_k(dir d)  of direction
// d into terms[d][n], one block of 128 threads per direction.  W(k, n) = w[k sk + n sn] over nk encoding elements of
// num_deg degrees: the packed image's [27][128] (the tensor-core precisions; the fmaf order of level_view_terms, so
// each term is radiance mode's bit for bit) or view_layers.0's own columns (fp32).
__global__ void __launch_bounds__(kCond) view_terms_kernel(const float* __restrict__ dirs, const float* __restrict__ w,
                                                           int64_t sk, int64_t sn, const float* __restrict__ bias,
                                                           int nk, int num_deg, float* __restrict__ terms) {
  __shared__ float enc[kViewDim];
  const int64_t d = blockIdx.x;
  const int n = threadIdx.x;
  if (n < nk) enc[n] = view_enc_elem(dirs + d * 3, n, num_deg);
  __syncthreads();
  float acc = __ldg(bias + n);
  for (int k = 0; k < nk; ++k) acc = fmaf(__ldg(w + k * sk + n * sn), enc[k], acc);
  terms[d * kCond + n] = acc;
}

// The per-(point, direction) head: y = max(A[p] + T[d], 0) and the colour head on it in the level kernel's order (four
// partial sums, one per quad lane q over columns 8 j + 2 q, + 1 for j = 0..15; combined as quad_sum combines them; then
// b_color), so that raw_rgb is radiance mode's bit for bit.  One thread per point with its A row in registers; the
// terms, the table and W_color are broadcast from shared memory, kPairDirs directions at a time.  kProj: proj[p][k][ch] =
// sum over d = 0..D-1, in order, of table[d][k] c[p][d][ch] (c: raw_rgb when proj_raw, else rgb), in fp32.
constexpr int kPairThreads = 128;
constexpr int kPairDirs = 32;
constexpr int kMaxBasis = 16;
template <bool kProj>
__global__ void __launch_bounds__(kPairThreads) radiance_pairs_kernel(
    const float* __restrict__ acc, const float* __restrict__ terms, const float* __restrict__ w_color,
    const float* __restrict__ b_color, int64_t num_points, int64_t num_dirs, float rgb_scale, float rgb_padding,
    float* __restrict__ raw_rgb, float* __restrict__ rgb, const float* __restrict__ table, int num_basis, int proj_raw,
    float* __restrict__ proj) {
  __shared__ __align__(16) float s_w[3][kCond];
  __shared__ __align__(16) float s_t[kPairDirs][kCond];
  __shared__ float s_tab[kPairDirs][kMaxBasis];
  const int tid = threadIdx.x;
  const int64_t pt = (int64_t)blockIdx.x * kPairThreads + tid;
  const bool live = pt < num_points;
  for (int i = tid; i < 3 * kCond; i += kPairThreads) s_w[i / kCond][i % kCond] = __ldg(w_color + i);
  float a[kCond];
  const float4* ar = reinterpret_cast<const float4*>(acc + (live ? pt : 0) * kCond);
#pragma unroll
  for (int j = 0; j < kCond / 4; ++j) {
    const float4 v = __ldcs(ar + j);  // read once
    a[4 * j] = v.x, a[4 * j + 1] = v.y, a[4 * j + 2] = v.z, a[4 * j + 3] = v.w;
  }
  const float bc[3] = {__ldg(b_color), __ldg(b_color + 1), __ldg(b_color + 2)};
  float pr[kProj ? kMaxBasis : 1][3];
#pragma unroll
  for (int k = 0; k < (kProj ? kMaxBasis : 1); ++k) pr[k][0] = pr[k][1] = pr[k][2] = 0.f;
#pragma unroll 1
  for (int64_t d0 = 0; d0 < num_dirs; d0 += kPairDirs) {
    const int nd = (int)(num_dirs - d0 < kPairDirs ? num_dirs - d0 : kPairDirs);
    __syncthreads();  // the previous round's reads of s_t / s_tab are done
    for (int i = tid; i < nd * kCond; i += kPairThreads) s_t[i / kCond][i % kCond] = __ldg(terms + d0 * kCond + i);
    if (kProj)
      for (int i = tid; i < nd * kMaxBasis; i += kPairThreads) {
        const int dd = i / kMaxBasis, k = i % kMaxBasis;
        s_tab[dd][k] = k < num_basis ? __ldg(table + (d0 + dd) * num_basis + k) : 0.f;
      }
    __syncthreads();
    if (!live) continue;
#pragma unroll 1
    for (int dd = 0; dd < nd; ++dd) {
      // W_color re-read from shared memory per direction: opaque here, so that the compiler does not keep its 384
      // loop-invariant values in registers beside the A row (ptxas spills 1.6 KB otherwise)
      const float* wc = &s_w[0][0];
      asm volatile("" : "+l"(wc));
      float s[4][3];
#pragma unroll
      for (int q = 0; q < 4; ++q) s[q][0] = s[q][1] = s[q][2] = 0.f;
#pragma unroll
      for (int j = 0; j < kCond / 8; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * j + 2 * q + e;
            const float y = fmaxf(__fadd_rn(a[c], s_t[dd][c]), 0.f);
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) s[q][ch] = __fmaf_rn(y, wc[ch * kCond + c], s[q][ch]);
          }
      const int64_t o = (pt * num_dirs + d0 + dd) * 3;
      float cv[3];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float raw = __fadd_rn(__fadd_rn(__fadd_rn(s[0][ch], s[1][ch]), __fadd_rn(s[2][ch], s[3][ch])), bc[ch]);
        const float act = rgb_activation(raw, rgb_scale, rgb_padding);
        if (raw_rgb) raw_rgb[o + ch] = raw;
        if (rgb) rgb[o + ch] = act;
        cv[ch] = proj_raw ? raw : act;
      }
      if (kProj) {
#pragma unroll
        for (int k = 0; k < (kProj ? kMaxBasis : 1); ++k) {
          if (k >= num_basis) break;
          const float t = s_tab[dd][k];
#pragma unroll
          for (int ch = 0; ch < 3; ++ch) pr[k][ch] = __fmaf_rn(t, cv[ch], pr[k][ch]);
        }
      }
    }
  }
  if (kProj && live) {
#pragma unroll
    for (int k = 0; k < (kProj ? kMaxBasis : 1); ++k) {
      if (k >= num_basis) break;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) proj[(pt * num_basis + k) * 3 + ch] = pr[k][ch];
    }
  }
}

// ---- weight packing ---------------------------------------------------------------------------
// lo != 0: the low half  fl16(w - fl16(w))  of the split-operand modes instead of fl16(w)
template <int kFmt>
__global__ void pack_stage_kernel(const float* __restrict__ w, int in_features, int row0, int kbase, int kcount,
                                  uint8_t* __restrict__ dst, int nrows, int lo) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nrows * kcount) return;
  const int i = idx / kcount, j = idx % kcount;
  float v = w[(size_t)(row0 + i) * in_features + kbase + j];
  if (lo) v = v - from16<kFmt>(to16<kFmt>(v));
  const uint32_t off = kcount == 64 ? sw128_offset(i, j) : sw64_offset(i, j);
  *reinterpret_cast<uint16_t*>(dst + off) = to16<kFmt>(v);
}

// All stages of one (hi or lo) v1 image in ONE launch: block = stage.  Stage (layer l, N-half h, K-slab s) as w_stage
// lays it out (K order of layer 5 is the reference's concat [h (256) | x (96)], mip_nerf.py:96-97): [128 x kw] at K
// offset k0, SW128 for 64-wide stages, SW64 for 32-wide ones.
struct PackV1Src {
  const float* weight[kNumLayers];
  int in_features[kNumLayers];
};
__host__ __device__ constexpr int v1_stage_begin(bool wide, int l) {
  int n = 0;
  for (int i = 0; i < l; ++i) n += num_halves(i) * num_slabs(wide, i);
  return n;
}
template <int kFmt>
__global__ void __launch_bounds__(256) pack_v1_image_kernel(const PackV1Src src, uint8_t* __restrict__ base, int lo,
                                                            bool wide) {
  const int stage = blockIdx.x;
  int l = 0;
  while (l + 1 < kNumLayers && stage >= v1_stage_begin(wide, l + 1)) ++l;
  const int local = stage - v1_stage_begin(wide, l);
  const int h = local / num_slabs(wide, l), sl = local % num_slabs(wide, l);
  const WStage ws = w_stage(wide, l, sl);
  const float* w = src.weight[l];
  const int in_features = src.in_features[l], row0 = h * 128, nrows = 128;
  uint8_t* dst = base + w_stage_offset(wide, l, h, sl);
  for (int idx = threadIdx.x; idx < nrows * ws.kw; idx += 256) {
    const int i = idx / ws.kw, j = idx % ws.kw;
    float v = w[(size_t)(row0 + i) * in_features + ws.k0 + j];
    if (lo) v = v - from16<kFmt>(to16<kFmt>(v));
    *reinterpret_cast<uint16_t*>(dst + (ws.sw128 ? sw128_offset(i, j) : sw64_offset(i, j))) = to16<kFmt>(v);
  }
}

// dst [rows, in_dst] <- src [rows, in_src]: the first `prefix` columns copied; the rest is two halves (sin | shifted sin)
// of half_dst columns each, of which the model has the first half_src (lower encoding degrees); the others are zero
__global__ void expand_encoding_columns_kernel(const float* __restrict__ src, int in_src, float* __restrict__ dst,
                                               int in_dst, int rows, int prefix, int half_src, int half_dst) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * in_dst) return;
  const int r = idx / in_dst, c = idx % in_dst;
  float v = 0.f;
  if (c < prefix) {
    v = src[(size_t)r * in_src + c];
  } else {
    const int j = c - prefix, h = j / half_dst, i = j % half_dst;
    if (h < 2 && i < half_src) v = src[(size_t)r * in_src + prefix + h * half_src + i];
  }
  dst[idx] = v;
}

struct SmallSrc {
  const float* bias[9];
  const float* w_density;
  const float* b_density;
  const float* w_color;
  const float* b_color;
};
__global__ void pack_small_params_kernel(const SmallSrc src, SmallParams* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 9 * kWidth) out->bias[i / kWidth][i % kWidth] = src.bias[i / kWidth][i % kWidth];
  if (i < kWidth) out->w_density[i] = src.w_density[i];
  if (i < 3 * kCond) out->w_color[i / kCond][i % kCond] = src.w_color[i];
  if (i == 0) out->b_density = src.b_density[0];
  if (i < 3) out->b_color[i] = src.b_color[i];
}

__global__ void pack_view_dir_kernel(const float* __restrict__ w, const float* __restrict__ b,
                                     float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kViewDim * kCond) {
    const int k = i / kCond, n = i % kCond;
    out[i] = w[(size_t)n * (kWidth + kViewDim) + kWidth + k];
  } else if (i < (kViewDim + 1) * kCond) {
    out[i] = b[i - kViewDim * kCond];
  }
}

// c_small is ONE constant bank per device, while the ABI lets callers run forwards of different models on different
// streams.  SmallUpload serialises those users: it holds a host lock for the duration of the enqueue, makes the
// stream wait for the previous user's kernels (on another stream) before overwriting the bank, and records an event
// after this call's launches.  Same-stream callers (the normal case) pay one event record.  During stream capture the
// cross-stream wait is skipped (a capture is single-stream by construction and the event lives outside the graph).
struct SmallBankState {
  cudaEvent_t done = nullptr;
  cudaStream_t last = nullptr;
  bool used = false;
};
std::mutex g_small_mu;
SmallBankState g_small_state[kMaxDevices];

class SmallUpload {
 public:
  SmallUpload(const uint8_t* img, cudaStream_t st) : lock_(g_small_mu), st_(st) {
    int dev = 0;
    cudaGetDevice(&dev);
    state_ = &g_small_state[dev % kMaxDevices];
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cap) != cudaSuccess) cap = cudaStreamCaptureStatusNone;
    capturing_ = cap != cudaStreamCaptureStatusNone;
    if (!capturing_ && state_->used && state_->last != st) {
      err_ = cudaStreamWaitEvent(st, state_->done, 0);
      if (err_ != cudaSuccess) return;
    }
    err_ = cudaMemcpyToSymbolAsync(c_small, img + kSmallOffset, sizeof(SmallParams), 0, cudaMemcpyDeviceToDevice, st);
  }
  cudaError_t error() const { return err_; }
  ~SmallUpload() {
    if (capturing_ || err_ != cudaSuccess) return;
    if (!state_->done && cudaEventCreateWithFlags(&state_->done, cudaEventDisableTiming) != cudaSuccess) return;
    if (cudaEventRecord(state_->done, st_) == cudaSuccess) {
      state_->last = st_;
      state_->used = true;
    }
  }

 private:
  std::lock_guard<std::mutex> lock_;
  cudaStream_t st_;
  SmallBankState* state_ = nullptr;
  bool capturing_ = false;
  cudaError_t err_ = cudaSuccess;
};

struct TcScratch {
  float *vbias, *t[2], *w[2];
  size_t bytes;
};
// rays per launch of the level kernels: 65536 at 128 samples, 32768 at 256 (the same scratch per chunk, and still
// 500 rays per SM)
constexpr int64_t kChunkRaysTc = 65536;
inline int64_t tc_chunk_rays(int n) { return kChunkRaysTc * kN / n; }

TcScratch carve_tc(int64_t rays, int n, void* base) {
  TcScratch s{};
  Carver cv{base};
  s.vbias = cv.floats((size_t)rays * kCond);
  for (int i = 0; i < 2; ++i) {
    s.t[i] = cv.floats((size_t)rays * (n + 1));
    s.w[i] = cv.floats((size_t)rays * n);
  }
  s.bytes = cv.off;
  return s;
}

template <int kFmt, bool kX3, int kT, int kMode = kModeForward, bool kTrain = false, bool kQueryDump = false>
cudaError_t launch_level_t(const LevelParams& p, cudaStream_t st) {
  constexpr auto kern = mlp_level_kernel<kFmt, kX3, kT, kMode, kTrain, kQueryDump>;
  constexpr uint32_t smem = LevelLayout<kX3, kT>::kTotal;
  cudaError_t e = allow_smem<kern>((int)smem);
  if (e != cudaSuccess) return e;
  int sms = 0;
  if ((e = num_sms(&sms)) != cudaSuccess) return e;
  LaunchScope scope(kMode == kModeDensity    ? kKernDensityTc
                    : kMode == kModeRadiance ? kKernRadianceTc
                    : kMode == kModeViewAcc  ? kKernRadianceDirsTc
                                             : (p.feat_in ? kKernMlpTc : kKernMlpLevelTc),
                    st);
  const int grid = (int)(p.num_rays < sms ? p.num_rays : sms);
  kern<<<grid, kThreads, smem, st>>>(p);
  return cudaGetLastError();
}

// One launch of the level kernel in mode kMode with kT 128-row tiles per ray (n = 128 or 256 samples per ray), on the
// operand format and split of `precision`.  A query's backward (p.act_dump in density / radiance mode) takes the query
// dump variant, which exists for bf16 / fp16 only; the training forward of the split precisions is tc_forward's.
template <int kMode, int kT = 1>
cudaError_t launch_level(const LevelParams& p, int precision, cudaStream_t st) {
  if (p.num_rays <= 0) return cudaSuccess;
  const bool bf = fmt_of(precision) == MIPNERF_B200_BF16;
  if constexpr (kMode == kModeDensity || kMode == kModeRadiance)
    if (p.act_dump)
      return bf ? launch_level_t<1, false, 1, kMode, false, true>(p, st)
                : launch_level_t<0, false, 1, kMode, false, true>(p, st);
  if (is_x3(precision))
    return bf ? launch_level_t<1, true, kT, kMode>(p, st) : launch_level_t<0, true, kT, kMode>(p, st);
  return bf ? launch_level_t<1, false, kT, kMode>(p, st) : launch_level_t<0, false, kT, kMode>(p, st);
}

// The launch parameters every query mode shares: points [off, off + cnt) of the query's Gaussians as tiles of 128
// points, their density outputs (either may be null) and, for a query's backward, the dump.
LevelParams query_params(const mipnerf_b200_config* c, const uint8_t* img, const float* means, const float* covs,
                         int64_t off, int64_t cnt, float* raw_density, float* density, const TcQueryDump* dump) {
  LevelParams p{};
  p.wimage = img;
  p.q_means = means + off * 3;
  p.q_covs = covs ? covs + off * 3 : nullptr;
  p.num_points = cnt;
  p.num_rays = (cnt + kN - 1) / kN;
  p.raw_density_out = raw_density ? raw_density + off : nullptr;
  p.density_out = density ? density + off : nullptr;
  p.disable_integration = c->disable_integration;
  p.density_bias = c->density_bias;
  if (dump) p.act_dump = dump->act, p.v_dump = dump->v, p.dump_tiles = p.num_rays;
  return p;
}

// radiance mode: the view-direction slots [ctas][2][128][128] fp32, one pair per CTA of a launch of min(tiles, SMs)
// (0 without a device)
constexpr size_t kRadianceSlotBytes = 2 * (size_t)kN * kCond * sizeof(float);
int64_t radiance_ctas(int64_t num_points) {
  const int64_t tiles = (num_points + kN - 1) / kN, chunk = kDensityChunkPoints / kN;
  const int64_t t = tiles < chunk ? tiles : chunk;
  int sms = 0;
  num_sms(&sms);
  return t < sms ? t : sms;
}

}  // namespace

// Encoding degrees below the kernels' own (max_deg_point < 16, deg_view < 4; min_deg_point = 0): the level kernels always
// compute the 96 IPE features of degrees 0..15 and the 27 view features of degrees 0..3, and the MODEL's narrower
// layers.0 / layers.5 / view_layers.0 weights are zero-padded to those widths when the operand image is packed (feature
// column 3 l + c of the sin half and 48 + 3 l + c of the shifted-sin half <- the model's columns 3 l + c and
// 3 L + 3 l + c; models/mip.py:322-341, :353-363).  The extra features meet exact zeros in the GEMM, so the result is the
// narrower model's, at the default model's speed.
bool tc_default_degrees(const mipnerf_b200_config* c) { return c->max_deg_point == 16 && c->deg_view == 4; }
bool tc_supported(const mipnerf_b200_config* c, int precision) {
  return (precision == MIPNERF_B200_BF16 || precision == MIPNERF_B200_FP16 || is_x3(precision)) &&
         (c->num_samples == kN || c->num_samples == 2 * kN) &&
         c->min_deg_point == 0 && c->max_deg_point >= 1 && c->max_deg_point <= 16 && c->deg_view >= 1 &&
         c->deg_view <= 4 && c->use_viewdirs &&
         c->net_depth == 8 && c->net_width == kWidth && c->net_depth_condition == 1 &&
         c->net_width_condition == kCond && c->skip_index == 4 && c->num_rgb_channels == 3 &&
         c->num_density_channels == 1;
}
bool tc_mlp_supported(const mipnerf_b200_config* c, int samples_per_ray, int precision) {
  mipnerf_b200_config c2 = *c;
  c2.num_samples = kN;  // MLP-only mode takes the caller's [B,128,96] / [B,27] encodings as they are: default degrees only
  return samples_per_ray == kN && tc_default_degrees(c) && tc_supported(&c2, precision);
}

// zero-padded fp32 copies of layers.0 [256,96], layers.5 [256,352], view_layers.0 [128,283] behind the operand image
constexpr size_t kPad0Bytes = (size_t)kWidth * kFeat * sizeof(float);
constexpr size_t kPad5Bytes = (size_t)kWidth * (kWidth + kFeat) * sizeof(float);
constexpr size_t kPadViewBytes = (size_t)kCond * (kWidth + kViewDim) * sizeof(float);
constexpr size_t kPadOffset = (kImageEnd + 255) / 256 * 256;
constexpr size_t kPadBytes = kPad0Bytes + kPad5Bytes + kPadViewBytes;

size_t tc_packed_bytes(const mipnerf_b200_config* c, int precision) {
  if (!tc_supported(c, precision)) return 0;
  return tc_default_degrees(c) ? kImageEnd : kPadOffset + kPadBytes;
}

size_t tc_workspace_bytes(const mipnerf_b200_config* c, int64_t num_rays, int precision) {
  if (!tc_supported(c, precision)) return 0;
  return carve_tc(std::clamp<int64_t>(num_rays, 1, tc_chunk_rays(c->num_samples)), c->num_samples, nullptr).bytes;
}

cudaError_t tc_pack_weights(const mipnerf_b200_config* c, const mipnerf_b200_weights* w, int precision,
                            void* packed_out, cudaStream_t st) {
  if (!tc_supported(c, precision)) return cudaErrorNotSupported;
  uint8_t* img = static_cast<uint8_t*>(packed_out);
  const bool bf = fmt_of(precision) == MIPNERF_B200_BF16;
  const int parts = is_x3(precision) ? 2 : 1;  // hi image, then (split modes) the lo stage image
  cudaError_t e = cudaMemsetAsync(img, 0, kImageEnd, st);
  if (e != cudaSuccess) return e;
  LaunchScope scope(kKernPackWeights, st);
  mipnerf_b200_linear lin[12];
  for (int i = 0; i < 12; ++i) lin[i] = w->linears[i];
  if (!tc_default_degrees(c)) {  // lower encoding degrees: pack from zero-padded copies of the three encoding-fed layers
    float* pad0 = reinterpret_cast<float*>(img + kPadOffset);
    float* pad5 = reinterpret_cast<float*>(img + kPadOffset + kPad0Bytes);
    float* padv = reinterpret_cast<float*>(img + kPadOffset + kPad0Bytes + kPad5Bytes);
    const int hx = 3 * c->max_deg_point, hv = 3 * c->deg_view;
    auto expand = [&](int li, float* dst, int in_dst, int rows, int prefix, int half_src, int half_dst) {
      expand_encoding_columns_kernel<<<(rows * in_dst + 255) / 256, 256, 0, st>>>(lin[li].weight, lin[li].in_features, dst,
                                                                                  in_dst, rows, prefix, half_src, half_dst);
      lin[li].weight = dst, lin[li].in_features = in_dst;
    };
    expand(0, pad0, kFeat, kWidth, 0, hx, kFeat / 2);
    expand(5, pad5, kWidth + kFeat, kWidth, kWidth, hx, kFeat / 2);
    expand(10, padv, kWidth + kViewDim, kCond, kWidth + 3, hv, (kViewDim - 3) / 2);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  PackV1Src v1{};
  for (int l = 0; l < kNumLayers; ++l) {
    const int li = l < 8 ? l : (l == 8 ? 9 : 10);  // layers.l | extra_layer | view_layers.0
    v1.weight[l] = lin[li].weight, v1.in_features[l] = lin[li].in_features;
  }
  const bool wide = !is_x3(precision);  // the stage layout the level kernel of this precision streams
  const int stages = v1_stage_begin(wide, kNumLayers);
  for (int part = 0; part < parts; ++part) {
    uint8_t* base = img + (part ? kLoOffset : 0);
    if (bf) pack_v1_image_kernel<1><<<stages, 256, 0, st>>>(v1, base, part, wide);
    else pack_v1_image_kernel<0><<<stages, 256, 0, st>>>(v1, base, part, wide);
  }
  SmallSrc src;
  for (int l = 0; l < 8; ++l) src.bias[l] = lin[l].bias;
  src.bias[8] = lin[9].bias;  // extra_layer
  src.w_density = lin[8].weight;
  src.b_density = lin[8].bias;
  src.w_color = lin[11].weight;
  src.b_color = lin[11].bias;
  pack_small_params_kernel<<<(9 * kWidth + 255) / 256, 256, 0, st>>>(src,
                                                                      reinterpret_cast<SmallParams*>(img + kSmallOffset));
  pack_view_dir_kernel<<<((kViewDim + 1) * kCond + 255) / 256, 256, 0, st>>>(
      lin[10].weight, lin[10].bias, reinterpret_cast<float*>(img + kViewDirOffset));
  return cudaGetLastError();
}

// The uniforms of one launch: rows `off..` of the caller's array, or the in-kernel generator (stream 0 = t_rand,
// 1 + level = that level's u_jitter, scaled like uniform_(to = 1/ncols - eps), models/mip.py:201-202).
Draws level_draws(int randomized, const float* array, const mipnerf_b200_rng* rng, int64_t off, int stream, int ncols) {
  if (!randomized) return draws_from_array(nullptr);
  if (array) return draws_from_array(array + off * ncols);
  if (!rng) return draws_from_array(nullptr);
  const float scale = stream == 0 ? 1.0f : (float)(1.0 / (double)ncols) - MIPNERF_F32_EPS;
  return draws_philox(rng->seed, rng->offset, off, stream, scale);
}

// The density-noise normals of one launch of level `level` (models/mip_nerf.py:232-233): rows `off..` of the caller's
// [B,n] array, or the in-kernel generator (stream 32 + level); inactive unless randomized and density_noise > 0.
Draws density_noise_draws(const mipnerf_b200_config* c, int randomized, const float* normal, const mipnerf_b200_rng* rng,
                          int64_t off, int level, int n) {
  if (!randomized || !(c->density_noise > 0.f)) return draws_from_array(nullptr);
  Draws d = normal ? draws_from_array(normal + off * n)
                   : (rng ? draws_philox(rng->seed, rng->offset, off, kDensityNoiseStream + level, 1.f)
                          : draws_from_array(nullptr));
  d.scale = c->density_noise;
  return d;
}

cudaError_t tc_forward(const mipnerf_b200_config* c, const mipnerf_b200_weights* w, const mipnerf_b200_rays* rays,
                       int randomized, const float* t_rand, const float* u_jitter, const mipnerf_b200_rng* rng,
                       int white_bkgd, int precision, mipnerf_b200_level_out* outs, void* workspace,
                       size_t workspace_bytes, cudaStream_t st, const TcTrainDump* dump, int64_t ray_base,
                       int given_t, const float* const* proposal) {
  const uint8_t* img = static_cast<const uint8_t*>(w->packed);
  SmallUpload small(img, st);  // biases / heads -> constant bank, ordered against other streams' forwards
  cudaError_t e = small.error();
  if (e != cudaSuccess) return e;
  const float rgb_scale = rgb_scale_of(c);
  const int n = c->num_samples;
  const int64_t chunk = tc_chunk_rays(n);
  if (dump && n != kN) return cudaErrorNotSupported;  // the training dump is one tile per ray
  for (int64_t off = 0; off < rays->num_rays; off += chunk) {
    const int64_t cnt = (rays->num_rays - off) < chunk ? (rays->num_rays - off) : chunk;
    const TcScratch s = carve_tc(cnt, n, workspace);
    if (s.bytes > workspace_bytes) return cudaErrorInvalidValue;
    const float* origins = rays->origins + off * 3;
    const float* directions = rays->directions + off * 3;
    const float* radii = rays->radii + off;
    // in-kernel Philox: the counter is the ray index of the caller's whole batch (ray_base = offset of `rays` in it)
    auto draws = [&](const float* array, int stream) {
      Draws d = level_draws(randomized, array, rng, off, stream, n + 1);
      if (!array) d.ray_base += ray_base;
      return d;
    };
    const int first = proposal ? 1 : 0;
    const float* t_prev = proposal ? proposal[0] + off * (n + 1) : nullptr;
    const float* w_prev = proposal ? proposal[1] + off * n : nullptr;
    for (int l = first; l < c->num_levels; ++l) {
      const mipnerf_b200_level_out& o = outs[l - first];
      float* t_cur = o.t_samples ? o.t_samples + off * (n + 1) : s.t[l & 1];
      float* w_cur = o.weights ? o.weights + off * n : s.w[l & 1];
      const Draws jit = draws(u_jitter, 1 + l);  // one stream per level
      int64_t* inds = o.inds ? o.inds + off * (n + 1) : nullptr;
      LevelParams p{};
      p.wimage = img;
      p.origins = origins, p.directions = directions, p.radii = radii;
      p.t = t_cur;
      p.view_bias = s.vbias;
      p.t_mode = given_t ? 0 : (l == 0 ? 1 : 2);  // 0: the caller's fenceposts in outs[l].t_samples
      p.vb_mode = l == first ? 1 : 0;  // the first level leaves the per-ray bias in s.vbias for the later levels
      p.near = rays->near + off, p.far = rays->far + off;
      p.t_rand = draws(t_rand, 0);
      p.disparity = c->disparity;
      p.t_prev = t_prev, p.w_prev = w_prev;
      p.u_jitter = jit;
      p.inds = inds;
      p.randomized = randomized;
      p.resample_padding = c->resample_padding;
      p.viewdirs = rays->viewdirs + off * 3;
      if (dump) {  // training forward: one chunk only (the caller chunks), tile index = ray index
        p.act_dump = dump->act[l], p.v_dump = dump->v[l];
        p.raw_rgb_keep = dump->raw_rgb[l], p.raw_density_keep = dump->raw_density[l];
        p.dump_tiles = cnt;
      }
      p.comp_rgb = o.comp_rgb + off * 3;
      p.distance = o.distance + off;
      p.acc = o.acc + off;
      p.weights = w_cur;
      p.num_rays = cnt;
      p.white_bkgd = white_bkgd;
      p.disable_integration = c->disable_integration;
      p.density_bias = c->density_bias, p.rgb_scale = rgb_scale, p.rgb_padding = c->rgb_padding;
      p.dnoise = density_noise_draws(c, randomized, o.density_normal, rng, off, l, n);
      if (!o.density_normal) p.dnoise.ray_base += ray_base;
      // the split precisions' training forward dumps the lo halves as well (kTrain); bf16x3 is the one that trains
      if (dump && is_x3(precision))
        e = fmt_of(precision) == MIPNERF_B200_BF16 ? launch_level_t<1, true, 1, kModeForward, true>(p, st)
                                                  : cudaErrorNotSupported;
      else
        e = n == 2 * kN ? launch_level<kModeForward, 2>(p, precision, st)
                        : launch_level<kModeForward>(p, precision, st);
      if (e != cudaSuccess) return e;
      t_prev = t_cur;
      w_prev = w_cur;
    }
  }
  return cudaSuccess;
}

cudaError_t tc_mlp_forward(const mipnerf_b200_config* c, const mipnerf_b200_weights* w, const float* x,
                           const float* view_enc, int64_t num_rays, int precision, float* raw_rgb, float* raw_density,
                           void* workspace, cudaStream_t st) {
  (void)c;
  const uint8_t* img = static_cast<const uint8_t*>(w->packed);
  SmallUpload small(img, st);
  cudaError_t e = small.error();
  if (e != cudaSuccess) return e;
  float* vbias = static_cast<float*>(workspace);  // [num_rays, 128]
  const mipnerf_b200_linear& view = w->linears[10];
  {
    LaunchScope scope(kKernPosEnc, st);
    view_bias_from_enc_kernel<<<(unsigned)((num_rays * kCond + 255) / 256), 256, 0, st>>>(view_enc, view.weight,
                                                                                           view.bias, vbias, num_rays);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  LevelParams p{};
  p.wimage = img;
  p.view_bias = vbias;
  p.feat_in = x;
  p.raw_rgb_out = raw_rgb;
  p.raw_density_out = raw_density;
  p.num_rays = num_rays;
  return launch_level<kModeForward>(p, precision, st);
}

cudaError_t tc_query_density(const mipnerf_b200_config* c, const mipnerf_b200_weights* w, const float* means,
                             const float* covs, int64_t num_points, int precision, float* raw_density, float* density,
                             cudaStream_t st, const TcQueryDump* dump) {
  if (dump && (is_x3(precision) || num_points > kDensityChunkPoints)) return cudaErrorInvalidValue;
  const uint8_t* img = static_cast<const uint8_t*>(w->packed);
  SmallUpload small(img, st);
  cudaError_t e = small.error();
  if (e != cudaSuccess) return e;
  for (int64_t off = 0; off < num_points; off += kDensityChunkPoints) {
    const int64_t cnt = (num_points - off) < kDensityChunkPoints ? (num_points - off) : kDensityChunkPoints;
    const LevelParams p = query_params(c, img, means, covs, off, cnt, raw_density, density, dump);
    if ((e = launch_level<kModeDensity>(p, precision, st)) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

size_t tc_radiance_workspace_bytes(int64_t num_points) {
  return (size_t)radiance_ctas(num_points > 0 ? num_points : 1) * kRadianceSlotBytes;
}

cudaError_t tc_query_radiance(const mipnerf_b200_config* c, const mipnerf_b200_weights* w, const float* means,
                              const float* covs, const float* viewdirs, int64_t num_points, int precision,
                              float* raw_rgb, float* raw_density, float* rgb, float* density, void* workspace,
                              size_t workspace_bytes, cudaStream_t st, const TcQueryDump* dump) {
  if (workspace_bytes < tc_radiance_workspace_bytes(num_points)) return cudaErrorInvalidValue;
  if (dump && (is_x3(precision) || num_points > kDensityChunkPoints)) return cudaErrorInvalidValue;
  const uint8_t* img = static_cast<const uint8_t*>(w->packed);
  SmallUpload small(img, st);
  cudaError_t e = small.error();
  if (e != cudaSuccess) return e;
  for (int64_t off = 0; off < num_points; off += kDensityChunkPoints) {
    const int64_t cnt = (num_points - off) < kDensityChunkPoints ? (num_points - off) : kDensityChunkPoints;
    LevelParams p = query_params(c, img, means, covs, off, cnt, raw_density, density, dump);
    p.viewdirs = viewdirs + off * 3;
    p.view_bias = static_cast<float*>(workspace);  // the per-CTA slots, reused launch after launch on `st`
    p.raw_rgb_out = raw_rgb ? raw_rgb + off * 3 : nullptr;
    p.rgb_out = rgb ? rgb + off * 3 : nullptr;
    p.rgb_scale = rgb_scale_of(c);
    p.rgb_padding = c->rgb_padding;
    if ((e = launch_level<kModeRadiance>(p, precision, st)) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_view_bias_from_enc(const float* venc, const float* w, const float* b, float* out,
                                      int64_t num_rays, cudaStream_t st) {
  if (num_rays == 0) return cudaSuccess;
  LaunchScope scope(kKernPosEnc, st);
  view_bias_from_enc_kernel<<<(unsigned)((num_rays * kCond + 255) / 256), 256, 0, st>>>(venc, w, b, out, num_rays);
  return cudaGetLastError();
}

size_t tc_mlp_workspace_bytes(int64_t num_rays) { return (size_t)(num_rays > 0 ? num_rays : 1) * kCond * sizeof(float); }

cudaError_t tc_query_view_acc(const mipnerf_b200_config* c, const mipnerf_b200_weights* w, const float* means,
                              const float* covs, int64_t num_points, int precision, float* view_acc,
                              float* raw_density, float* density, cudaStream_t st) {
  if (num_points > kDensityChunkPoints) return cudaErrorInvalidValue;
  const uint8_t* img = static_cast<const uint8_t*>(w->packed);
  SmallUpload small(img, st);
  cudaError_t e = small.error();
  if (e != cudaSuccess) return e;
  LevelParams p = query_params(c, img, means, covs, 0, num_points, raw_density, density, nullptr);
  p.view_acc = view_acc;
  return launch_level<kModeViewAcc>(p, precision, st);
}

cudaError_t tc_view_terms(const mipnerf_b200_weights* w, const float* dirs, int64_t num_dirs, float* terms,
                          cudaStream_t st) {
  const float* wt = reinterpret_cast<const float*>(static_cast<const uint8_t*>(w->packed) + kViewDirOffset);
  return launch_view_terms(dirs, num_dirs, wt, kCond, 1, wt + kViewDim * kCond, kViewDim, (kViewDim - 3) / 6, terms, st);
}

cudaError_t launch_view_terms(const float* dirs, int64_t num_dirs, const float* w, int64_t sk, int64_t sn,
                              const float* bias, int nk, int num_deg, float* terms, cudaStream_t st) {
  if (num_dirs == 0) return cudaSuccess;
  if (nk > kViewDim) return cudaErrorInvalidValue;
  LaunchScope scope(kKernPosEnc, st);
  view_terms_kernel<<<(unsigned)num_dirs, kCond, 0, st>>>(dirs, w, sk, sn, bias, nk, num_deg, terms);
  return cudaGetLastError();
}

cudaError_t launch_radiance_pairs(const float* acc, const float* terms, const float* w_color, const float* b_color,
                                  int64_t num_points, int64_t num_dirs, float rgb_scale, float rgb_padding,
                                  float* raw_rgb, float* rgb, const float* table, int num_basis, int proj_raw,
                                  float* proj, cudaStream_t st) {
  if (num_points == 0 || num_dirs == 0) return cudaSuccess;
  if (proj && (num_basis < 1 || num_basis > kMaxBasis || !table)) return cudaErrorInvalidValue;
  LaunchScope scope(kKernRadiancePairs, st);
  const unsigned grid = (unsigned)((num_points + kPairThreads - 1) / kPairThreads);
  if (proj)
    radiance_pairs_kernel<true><<<grid, kPairThreads, 0, st>>>(acc, terms, w_color, b_color, num_points, num_dirs,
                                                               rgb_scale, rgb_padding, raw_rgb, rgb, table, num_basis,
                                                               proj_raw, proj);
  else
    radiance_pairs_kernel<false><<<grid, kPairThreads, 0, st>>>(acc, terms, w_color, b_color, num_points, num_dirs,
                                                                rgb_scale, rgb_padding, raw_rgb, rgb, nullptr, 0, 0,
                                                                nullptr);
  return cudaGetLastError();
}

}  // namespace mipnerf

#ifdef MIPNERF_LEVEL_PHASES
// Instrumented builds only (tools/level_phases.py): copies the per-CTA phase cycles accumulated since the last call,
// [2 slots][ctas][4 roles][phases] as uint64, into `out` and zeroes them.  Returns the phase count, or -1 on error.
extern "C" int mipnerf_b200_level_phases(unsigned long long* out, int* ctas) {
  using namespace mipnerf;
  *ctas = kPhaseMaxCtas;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(out, g_level_phases, sizeof(g_level_phases)) != cudaSuccess) return -1;
  void* dev = nullptr;
  if (cudaGetSymbolAddress(&dev, g_level_phases) != cudaSuccess || cudaMemset(dev, 0, sizeof(g_level_phases)) != cudaSuccess)
    return -1;
  return kNumPhases;
}
#endif
