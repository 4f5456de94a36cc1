// ray_math.cuh — per-ray device math shared by every kernel on the path.
//
// Each function restates one piece of the reference's models/mip.py with the SAME fp32 operation
// order; the pieces that decide downstream bit patterns (fenceposts, Gaussian means, the
// resampler) use __f*_rn intrinsics so nvcc cannot contract them into FMAs (torch-CPU rounds every
// op; SURVEY.md §8c item 4).
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "draws.h"

namespace mipnerf {

#define MIPNERF_HALF_PI_F32 1.57079637050628662109375f  // fl32(0.5*pi) = 0x3FC90FDB (models/mip.py:350)
#define MIPNERF_F32_EPS 1.1920928955078125e-07f          // torch.finfo(float32).eps
// ---- coarse fenceposts (models/mip.py:143-160) -------------------------------------------------
__device__ __forceinline__ float coarse_t(float near, float far, float s, int disparity) {
  if (disparity) {
    // 1 / (1/near*(1-s) + 1/far*s)        (models/mip.py:150)
    const float a = __fmul_rn(__fdiv_rn(1.0f, near), __fsub_rn(1.0f, s));
    const float b = __fmul_rn(__fdiv_rn(1.0f, far), s);
    return __fdiv_rn(1.0f, __fadd_rn(a, b));
  }
  return __fadd_rn(near, __fmul_rn(__fsub_rn(far, near), s));  // near + (far-near)*s   (:153)
}

// torch.linspace(start, end, steps)[j] on CPU, float32: step = fl32((end-start)/(steps-1)); the first half counts up
// from `start`, the second half DOWN from `end`, each element rounded once (ATen evaluates start + step*j in double,
// which is exact before the final rounding, i.e. an fma).  For steps-1 a power of two both halves reduce to
// fl32(j*step); for the other sample counts (96, 192) the second half differs from j*step by an ulp.
__device__ __forceinline__ float linspace_f32(float start, float end, int steps, int j) {
  const float step = __fdiv_rn(__fsub_rn(end, start), (float)(steps - 1));
  return j < steps / 2 ? __fmaf_rn(step, (float)j, start) : __fmaf_rn(-step, (float)(steps - 1 - j), end);
}

// ---- uniforms of randomized=True --------------------------------------------------------------------
// The reference draws them with torch.rand / uniform_ (models/mip.py:159, :201-202).  Here they come either from an
// explicit array (caller-injected noise: what the parity tests use to feed the reference's own draws) or from a
// counter-based generator evaluated inside the kernels that consume them: Philox4x32-10 keyed by `seed`, counter =
// (global ray index, draw index, stream, offset).  No state, no extra launch, no [B, N+1] array in HBM; draws do not
// depend on how the batch is chunked or sharded (ray_base) and are reproduced by mipnerf_b200_philox_uniform.
__device__ __forceinline__ uint32_t philox4x32_10_first(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                        uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}
// draw j of `ray` (row-local index): explicit array element, or scale * U[0,1) with 24 random bits
__device__ __forceinline__ float draw_uniform(const Draws& d, int64_t ray, int j, int ncols) {
  if (d.ptr) return __ldg(d.ptr + ray * ncols + j);
  const uint64_t g = (uint64_t)(d.ray_base + ray);
  const uint32_t x = philox4x32_10_first((uint32_t)g, (uint32_t)(g >> 32), (uint32_t)j | ((uint32_t)d.stream << 24),
                                         (uint32_t)d.offset, (uint32_t)d.seed,
                                         (uint32_t)(d.seed >> 32) ^ (uint32_t)(d.offset >> 32));
  return __fmul_rn((float)(x >> 8) * 5.9604644775390625e-08f, d.scale);  // 2^-24
}

// ---- density noise of randomized=True (models/mip_nerf.py:232-233: raw_density += density_noise * randn) ----------
// Standard normal j of `ray`: explicit array element (caller-injected draws, what the parity tests feed from the
// reference's own torch.randn), or Box-Muller on two 24-bit Philox uniforms of counter (ray, j, stream 32 + level).
__device__ __forceinline__ float draw_normal(const Draws& d, int64_t ray, int j, int ncols) {
  if (d.ptr) return __ldg(d.ptr + ray * ncols + j);
  const uint64_t g = (uint64_t)(d.ray_base + ray);
  const uint32_t k0 = (uint32_t)d.seed, k1 = (uint32_t)(d.seed >> 32) ^ (uint32_t)(d.offset >> 32);
  const uint32_t c2 = (uint32_t)j | ((uint32_t)d.stream << 24);
  const uint32_t x0 = philox4x32_10_first((uint32_t)g, (uint32_t)(g >> 32), c2, (uint32_t)d.offset, k0, k1);
  const uint32_t x1 = philox4x32_10_first((uint32_t)g, (uint32_t)(g >> 32), c2 | 0x800000u, (uint32_t)d.offset, k0, k1);
  const float u1 = (float)((x0 >> 8) + 1u) * 5.9604644775390625e-08f;  // (0, 1]
  const float u2 = (float)(x1 >> 8) * 5.9604644775390625e-08f;         // [0, 1)
  return __fmul_rn(sqrtf(__fmul_rn(-2.0f, logf(u1))), cospif(__fmul_rn(2.0f, u2)));
}
// raw density + scale * normal, mul and add rounded separately like the reference's two torch ops
__device__ __forceinline__ float add_density_noise(float raw_density, const Draws& d, int64_t ray, int j, int ncols) {
  return __fadd_rn(raw_density, __fmul_rn(d.scale, draw_normal(d, ray, j, ncols)));
}

// fencepost j of n+1; `jit` = t_rand[ray][j] for the stratified draw when has_jitter, ignored otherwise
__device__ __forceinline__ float coarse_fencepost(float nr, float fr, int j, int n, int disparity, bool has_jitter,
                                                  float jit) {
  float t = coarse_t(nr, fr, linspace_f32(0.0f, 1.0f, n + 1, j), disparity);  // models/mip.py:143
  if (has_jitter) {
    // mids / upper / lower (models/mip.py:156-160)
    const float lower =
        j == 0 ? t : __fmul_rn(0.5f, __fadd_rn(t, coarse_t(nr, fr, linspace_f32(0.0f, 1.0f, n + 1, j - 1), disparity)));
    const float upper =
        j == n ? t : __fmul_rn(0.5f, __fadd_rn(coarse_t(nr, fr, linspace_f32(0.0f, 1.0f, n + 1, j + 1), disparity), t));
    t = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), jit));
  }
  return t;
}


struct RayGeom {
  float o[3];     // origin
  float d[3];     // direction (not normalised)
  float d_sq[3];  // d*d                     (models/mip.py:29)
  float null[3];  // 1 - d*d/(sum d*d+1e-10) (models/mip.py:30)
  float radius_sq;
};

__device__ __forceinline__ RayGeom load_ray_geom(const float* __restrict__ origins,
                                                 const float* __restrict__ directions,
                                                 const float* __restrict__ radii, int64_t ray) {
  RayGeom g;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    g.o[c] = __ldg(origins + ray * 3 + c);
    g.d[c] = __ldg(directions + ray * 3 + c);
    g.d_sq[c] = __fmul_rn(g.d[c], g.d[c]);
  }
  // torch.sum over 3 contiguous elements is sequential; + float32(1e-10)  (models/mip.py:25)
  float dn = __fadd_rn(__fadd_rn(__fadd_rn(g.d_sq[0], g.d_sq[1]), g.d_sq[2]), 1e-10f);
#pragma unroll
  for (int c = 0; c < 3; ++c) g.null[c] = __fsub_rn(1.0f, __fdiv_rn(g.d_sq[c], dn));
  float r = __ldg(radii + ray);
  g.radius_sq = __fmul_rn(r, r);
  return g;
}

// conical_frustum_to_gaussian, stable branch (models/mip.py:65-72).
__device__ __forceinline__ void frustum_moments(float t0, float t1, float radius_sq, float& t_mean,
                                                float& t_var, float& r_var) {
  const float mu = __fmul_rn(__fadd_rn(t0, t1), 0.5f);
  const float hw = __fmul_rn(__fsub_rn(t1, t0), 0.5f);
  const float mu2 = __fmul_rn(mu, mu);
  const float hw2 = __fmul_rn(hw, hw);
  const float hw4 = __fmul_rn(hw2, hw2);  // reference: pow(hw,4) (<=1 ulp away; feeds variances only)
  const float denom = __fadd_rn(__fmul_rn(3.0f, mu2), hw2);
  t_mean = __fadd_rn(mu, __fdiv_rn(__fmul_rn(__fmul_rn(2.0f, mu), hw2), denom));
  const float c415 = 0.26666666666666666f;  // float32(4/15)
  const float num = __fmul_rn(hw4, __fsub_rn(__fmul_rn(12.0f, mu2), hw2));
  t_var = __fsub_rn(__fdiv_rn(hw2, 3.0f),
                    __fmul_rn(c415, __fdiv_rn(num, __fmul_rn(denom, denom))));
  const float c512 = 0.4166666666666667f;  // float32(5/12)
  const float a = __fadd_rn(__fdiv_rn(mu2, 4.0f), __fmul_rn(c512, hw2));
  const float b = __fdiv_rn(__fmul_rn(c415, hw4), denom);
  r_var = __fmul_rn(radius_sq, __fsub_rn(a, b));
}

// lift_gaussian diagonal branch + origin shift (models/mip.py:24-36, :102).
__device__ __forceinline__ void lift_gaussian(const RayGeom& g, float t_mean, float t_var,
                                              float r_var, float mean[3], float cov[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    mean[c] = __fadd_rn(__fmul_rn(g.d[c], t_mean), g.o[c]);
    cov[c] = __fadd_rn(__fmul_rn(t_var, g.d_sq[c]), __fmul_rn(r_var, g.null[c]));
  }
}

// One IPE feature pair for coordinate value `m`, variance `v`, degree l (scale 2^l):
//   sin-half  exp(-0.5*v*4^l) * sin(m*2^l)
//   cos-half  exp(-0.5*v*4^l) * sin(fl32(m*2^l + fl32(pi/2)))        (models/mip.py:335-350,:286)
// When the damping factor underflows to exactly 0 the feature is +-0 for any finite sin(y), so the
// sine (and its slow large-argument path) is skipped — bit-identical up to the sign of zero, and NaN
// where the reference's sin(y) is NaN.
template <bool kFast>
__device__ __forceinline__ void ipe_pair(float m, float v, int l, float& f_sin, float& f_cos);

__device__ __forceinline__ float sin_reduced_fast(float x) {
  // 2-term Cody-Waite reduction to [-pi, pi] (exact under FMA for |x| < 2^18) + MUFU.SIN.
  const float k = rintf(x * 0.15915494309189535f);
  float r = fmaf(k, -6.283185482025146484375f, x);      // fl32(2*pi)
  r = fmaf(k, 1.7484555e-07f, r);                       // 2*pi - fl32(2*pi) = -1.7484555e-07
  return __sinf(r);
}

template <>
__device__ __forceinline__ void ipe_pair<false>(float m, float v, int l, float& f_sin, float& f_cos) {
  const float scale = __int_as_float((127 + l) << 23);       // 2^l
  const float scale_sq = __int_as_float((127 + 2 * l) << 23);  // 4^l
  const float e_arg = __fmul_rn(-0.5f, __fmul_rn(v, scale_sq));
  const float y = __fmul_rn(m, scale);
  if (e_arg < -104.0f) {  // expf(x) == 0 for x < -103.98
    // the reference's 0 * sin(y) is NaN when y is NaN or infinite (a non-finite mean); +-0 otherwise
    f_sin = f_cos = isfinite(y) ? 0.0f : CUDART_NAN_F;
    return;
  }
  const float e = expf(e_arg);
  f_sin = __fmul_rn(e, sinf(y));
  f_cos = __fmul_rn(e, sinf(__fadd_rn(y, MIPNERF_HALF_PI_F32)));
}

template <>
__device__ __forceinline__ void ipe_pair<true>(float m, float v, int l, float& f_sin, float& f_cos) {
  // branch-free (8 pairs interleave): the damping factor is 2^(max(arg*log2e, -126)), i.e. <= 1.2e-38
  // where the reference underflows to 0 — far below the 16-bit operand rounding this path feeds.
  const float scale = __int_as_float((127 + l) << 23);
  const float scale_sq = __int_as_float((127 + 2 * l) << 23);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fmaxf(v * (scale_sq * -0.72134752044448170368f), -126.0f)));
  const float y = m * scale;
  f_sin = e * sin_reduced_fast(y);
  f_cos = e * sin_reduced_fast(__fadd_rn(y, MIPNERF_HALF_PI_F32));
}

// rgb = sigmoid(raw)*(1+2*pad) - pad ; density = softplus(raw + bias)   (models/mip_nerf.py:236-238)
// rgb_scale = float32(1 + 2*pad) is formed on the host in double like Python does.
__device__ __forceinline__ float rgb_activation(float raw, float rgb_scale, float rgb_padding) {
  const float s = 1.0f / (1.0f + expf(-raw));
  return __fsub_rn(__fmul_rn(s, rgb_scale), rgb_padding);
}
__device__ __forceinline__ float density_activation(float raw, float density_bias) {
  const float x = __fadd_rn(raw, density_bias);
  return x > 20.0f ? x : log1pf(expf(x));  // torch.nn.Softplus(beta=1, threshold=20)
}

// ---- warp helpers -------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_excl_scan_f64(double v, int lane, double& total) {
  double inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    double n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  total = __shfl_sync(0xffffffffu, inc, 31);
  double excl = __shfl_up_sync(0xffffffffu, inc, 1);
  return lane == 0 ? 0.0 : excl;
}

}  // namespace mipnerf
