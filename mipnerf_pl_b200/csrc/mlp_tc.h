// mlp_tc.h — internal interface of the wgmma (tensor-core) path, implemented in mlp_tc.cu.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <atomic>
#include <type_traits>

#include "../../include/mipnerf_b200.h"
#include "draws.h"

namespace mipnerf {

// 1 + 2 rgb_padding, the scale of the padded sigmoid colour activation (models/mip_nerf.py:236)
inline float rgb_scale_of(const mipnerf_b200_config* c) { return (float)(1.0 + 2.0 * (double)c->rgb_padding); }

// The 16-bit operand format of a tensor-core precision (MIPNERF_B200_BF16 or MIPNERF_B200_FP16) and whether the
// precision is split, carrying every operand as a hi / lo pair of that format.
inline int fmt_of(int precision) {
  return (precision == MIPNERF_B200_BF16 || precision == MIPNERF_B200_BF16X3) ? MIPNERF_B200_BF16 : MIPNERF_B200_FP16;
}
inline bool is_x3(int precision) { return precision == MIPNERF_B200_FP16X3 || precision == MIPNERF_B200_BF16X3; }

// Calls f(fmt, split) with the kernels' template arguments kFmt (1: bf16, 0: fp16, the format fmt_of(precision)) and
// kX3 = split as std::integral_constants, and returns what f returns.  The split (x3) variants of the launchers'
// kernels exist in bf16 only: split with fp16 is refused before f runs.
template <typename F>
cudaError_t with_fmt(int precision, bool split, F&& f) {
  using Bf16 = std::integral_constant<int, 1>;
  if (fmt_of(precision) == MIPNERF_B200_BF16) return split ? f(Bf16{}, std::true_type{}) : f(Bf16{}, std::false_type{});
  return split ? cudaErrorInvalidValue : f(std::integral_constant<int, 0>{}, std::false_type{});
}

// Devices with host state of their own (the caches below query a device past them every time).
constexpr int kMaxDevices = 64;

// The current device's SM count, queried once per device; *sms = 0 if the query fails.
inline cudaError_t num_sms(int* sms) {
  static std::atomic<int> cache[kMaxDevices];
  int dev = 0, n = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess && dev < kMaxDevices) n = cache[dev].load(std::memory_order_relaxed);
  if (e == cudaSuccess && n == 0) e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) n = 0;
  else if (dev < kMaxDevices) cache[dev].store(n, std::memory_order_relaxed);
  *sms = n;
  return e;
}

// Lets kKernel (one kernel instantiation) take `bytes` of dynamic shared memory on the current device, once per
// device.  Two threads racing here both set the same attribute, which is harmless.
template <auto kKernel>
cudaError_t allow_smem(int bytes) {
  static std::atomic<bool> done[kMaxDevices];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < kMaxDevices && done[dev].load(std::memory_order_relaxed)) return cudaSuccess;
  e = cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && dev < kMaxDevices) done[dev].store(true, std::memory_order_relaxed);
  return e;
}

inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

// The scratch layouts' bump allocator: 256-byte-aligned takes from `base` in call order; a null base only counts bytes.
struct Carver {
  void* base;
  size_t off = 0;
  uint8_t* bytes(size_t n) {
    uint8_t* p = base ? static_cast<uint8_t*>(base) + off : nullptr;
    off += align_up(n);
    return p;
  }
  float* floats(size_t n) { return reinterpret_cast<float*>(bytes(n * sizeof(float))); }
};

// true iff (cfg, precision) is the shape the fused tensor-core kernels are specialised for.
bool tc_supported(const mipnerf_b200_config* cfg, int precision);
bool tc_default_degrees(const mipnerf_b200_config* cfg);  // max_deg_point == 16 && deg_view == 4 (no weight padding)
bool tc_mlp_supported(const mipnerf_b200_config* cfg, int samples_per_ray, int precision);
size_t tc_packed_bytes(const mipnerf_b200_config* cfg, int precision);
size_t tc_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_rays, int precision);
cudaError_t tc_pack_weights(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, int precision,
                            void* packed_out, cudaStream_t st);
// Training forward: where the level kernels leave what the backward pass needs (per level l < 2; at most
// kTcTrainChunk rays per call).  Activations are 16-bit "tile images": per 128-row tile (= ray) and 64-column slab a
// [128 x 128 B] block in the 128-byte-swizzle layout the tensor core reads (sw128_offset), slabs of a tile contiguous.
struct TcTrainDump {
  uint8_t* act[2];        // [9][rays][64 KB]: h_0..h_7 (post-ReLU), bottleneck
  uint8_t* v[2];          // [rays][32 KB]: view-layer output (post-ReLU)
  float* raw_rgb[2];      // [rays,128,3]
  float* raw_density[2];  // [rays,128]
};
cudaError_t tc_forward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                       const mipnerf_b200_rays* rays, int randomized, const float* t_rand,
                       const float* u_jitter, const mipnerf_b200_rng* rng, int white_bkgd, int precision,
                       mipnerf_b200_level_out* outs, void* workspace, size_t workspace_bytes, cudaStream_t st,
                       const TcTrainDump* dump = nullptr, int64_t ray_base = 0, int given_t = 0,
                       const float* const* proposal = nullptr);
// given_t != 0: every level reads its fenceposts from outs[l].t_samples instead of generating them (sampling /
// resampling skipped; the backward pass of MipNerf.forward re-evaluates the MLP where the forward did)
// proposal = {t_prev [B,N+1], w_prev [B,N]}: the loop starts at level 1, resampling those in place of level 0's
// outputs; outs[l - 1] is level l's output, and level 1 computes the per-ray view bias level 0 would have
// the uniforms of one launch (see mlp_tc.cu)
Draws level_draws(int randomized, const float* array, const mipnerf_b200_rng* rng, int64_t off, int stream, int ncols);
// the density-noise normals of one launch of `level` (inactive unless randomized and cfg->density_noise > 0)
Draws density_noise_draws(const mipnerf_b200_config* cfg, int randomized, const float* normal,
                          const mipnerf_b200_rng* rng, int64_t off, int level, int n);
cudaError_t tc_mlp_forward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* x,
                           const float* view_enc, int64_t num_rays, int precision, float* raw_rgb,
                           float* raw_density, void* workspace, cudaStream_t st);
size_t tc_mlp_workspace_bytes(int64_t num_rays);
// Density-only mode of the level kernels (mipnerf_b200_query_density), kDensityChunkPoints points per launch; needs
// tc_supported(cfg, precision) and w->packed for that precision.
constexpr int64_t kDensityChunkPoints = 4096 * 128;
// The backward of a query: the query's tiles leave the training forward's dump (bf16 / fp16, at most one chunk of
// points per call; tile = query tile): act [layers][tiles][64 KB] with h_0..h_7 and, in radiance mode, the bottleneck;
// v [tiles][32 KB], the view-layer output (radiance mode).
struct TcQueryDump {
  uint8_t* act;
  uint8_t* v;
};
cudaError_t tc_query_density(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                             const float* covs, int64_t num_points, int precision, float* raw_density, float* density,
                             cudaStream_t st, const TcQueryDump* dump = nullptr);
// Radiance mode of the level kernels (mipnerf_b200_query_radiance), launched in the same chunks as the density query.
// The workspace is two [128][128] fp32 slots of view-direction terms per CTA of a launch, min(tiles, SMs) CTAs with
// tiles = ceil(points / 128) capped at one chunk's 4096.
size_t tc_radiance_workspace_bytes(int64_t num_points);
cudaError_t tc_query_radiance(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                              const float* covs, const float* viewdirs, int64_t num_points, int precision,
                              float* raw_rgb, float* raw_density, float* rgb, float* density, void* workspace,
                              size_t workspace_bytes, cudaStream_t st, const TcQueryDump* dump = nullptr);
// Radiance under a shared direction set (mipnerf_b200_query_radiance_dirs).  The view-accumulator mode of the level
// kernels, one launch for at most kDensityChunkPoints points: view_acc [ceil(points / 128) * 128][128] gets W_view[:, :256]
// . bottleneck of each point (the view layer's accumulators of radiance mode, before the view-direction term), raw_density
// / density (either may be null) the density query's values.
cudaError_t tc_query_view_acc(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                              const float* covs, int64_t num_points, int precision, float* view_acc,
                              float* raw_density, float* density, cudaStream_t st);
// terms [num_dirs][128]: radiance mode's view-direction term of each direction, from the packed image's view weights
cudaError_t tc_view_terms(const mipnerf_b200_weights* w, const float* dirs, int64_t num_dirs, float* terms,
                          cudaStream_t st);

}  // namespace mipnerf
