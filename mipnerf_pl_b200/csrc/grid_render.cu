// grid_render.cu — ray marching through a baked grid (mipnerf_b200_grid_render; the grid is built by
// mipnerf_pl_b200/baked.py, which owns the other half of the memory layout read here).
//
// One thread per ray, rays in the caller's (pixel) order, so that neighbouring threads walk neighbouring paths through
// the same cache lines.  Per ray:
//   * K, dt, t_k, delta and the sample positions o + t_k d are computed with explicitly rounded fp32 operations, so a
//     host restatement reproduces them exactly (tests/grid_render_ref.py).
//   * The sample range is first clipped to the bounds grown by a margin far above the rounding of those positions;
//     a sample outside the bounds has density 0, so clipping changes nothing.
//   * Inside, the macro cell of the sample is looked up in the occupancy grid.  An empty cell jumps k to the first
//     sample whose t is past the cell's exit t.  The occupancy builder marks a cell empty only when every level's
//     density is 0 on the cell's lattice points widened by one point of that level, so every skipped sample, and any
//     sample a rounding error away from the cell, interpolates to exactly 0 at every level: skipping is bit-exact.
//   * Density at the level(s) picked by the cone footprint is trilinear over the packed (density, SH row) lattice
//     points (one 8-byte load per corner).  Colour is evaluated only where the density is non-zero: each kept corner's
//     raw colour Y(viewdir) . c, blended with the corner weights and the level weights, then the model's sigmoid.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/mipnerf_b200.h"
#include "kernels.h"
#include "profile.h"

namespace mipnerf {
namespace {

constexpr int kGridThreads = 128;
constexpr float kStopTransmittance = 1e-4f;
constexpr float kSqrt3 = 1.7320508075688772f;

struct GLevel {
  const int2* cells;  // (density bits, SH row) per lattice point
  const float* sh;
  int n[3];
  float inv_s[3];  // (n - 1) / (hi - lo): lattice coordinate per unit length
};

struct GParams {
  GLevel lv[MIPNERF_B200_GRID_MAX_LEVELS];
  int num_levels, nc;  // nc = (degree + 1)^2
  float lo[3], hi[3];
  float s0[3];       // finest voxel edge per axis
  float s0_max;      // its largest
  float bound_mag;   // max |lo|, |hi|: scale of the clipping margin
  float rgb_scale, rgb_padding;
  const uint8_t* occ;
  int on[3];  // occupancy dims
  int block;
};

__device__ __forceinline__ float sample_t(float near, float dt, int64_t k) {
  return __fadd_rn(near, __fmul_rn(__fadd_rn((float)k, 0.5f), dt));
}

// The smallest k in [k0, k1] with t_k > thr (k1 if none), for dt > 0: t_k is non-decreasing in k, so an estimate is
// corrected by stepping against the exact fp32 t_k.
__device__ int64_t first_past(float thr, float near, float dt, int64_t k0, int64_t k1) {
  if (k0 >= k1 || !(thr >= sample_t(near, dt, k0))) return k0;
  if (thr >= sample_t(near, dt, k1 - 1)) return k1;
  const float e = floorf(__fsub_rn(__fdiv_rn(__fsub_rn(thr, near), dt), 0.5f)) + 1.f;
  int64_t k = e <= (float)(k0 + 1) ? k0 + 1 : e >= (float)(k1 - 1) ? k1 - 1 : (int64_t)e;
  while (k > k0 + 1 && sample_t(near, dt, k - 1) > thr) --k;
  while (sample_t(near, dt, k) <= thr) ++k;  // stops at k1 - 1 at the latest
  return k;
}

// Trilinear density of one level at position x: also the corner rows and weights, for the colour.
__device__ __forceinline__ float level_density(const GLevel& l, const float (&lo)[3], const float (&x)[3],
                                               int (&row)[8], float (&wc)[8]) {
  int i[3];
  float f[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float u = fminf(fmaxf((x[a] - lo[a]) * l.inv_s[a], 0.f), (float)(l.n[a] - 1));
    i[a] = min((int)u, l.n[a] - 2);
    f[a] = u - (float)i[a];
  }
  const int64_t base = ((int64_t)i[2] * l.n[1] + i[1]) * l.n[0] + i[0];
  const int64_t sy = l.n[0], sz = (int64_t)l.n[0] * l.n[1];
  float sigma = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
    const int2 v = __ldg(l.cells + base + dx + dy * sy + dz * sz);
    wc[c] = (dx ? f[0] : 1.f - f[0]) * (dy ? f[1] : 1.f - f[1]) * (dz ? f[2] : 1.f - f[2]);
    row[c] = v.y;
    sigma += wc[c] * __int_as_float(v.x);
  }
  return sigma;
}

// sum over kept corners of weight * Y . c (raw colour, 3 channels)
template <int NC>
__device__ __forceinline__ void level_color(const float* __restrict__ sh, const int (&row)[8], const float (&wc)[8],
                                            const float (&y)[16], float scale, float (&raw)[3]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (row[c] < 0) continue;
    const float* p = sh + (int64_t)row[c] * (NC * 3);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      s0 += y[k] * __ldg(p + 3 * k);
      s1 += y[k] * __ldg(p + 3 * k + 1);
      s2 += y[k] * __ldg(p + 3 * k + 2);
    }
    const float w = scale * wc[c];
    raw[0] += w * s0, raw[1] += w * s1, raw[2] += w * s2;
  }
}

// The (degree + 1)^2 real SH basis functions of field.sh_basis at unit direction (x, y, z).
__device__ __forceinline__ void sh_basis(float x, float y, float z, float (&b)[16]) {
  const float xx = x * x, yy = y * y, zz = z * z;
  b[0] = 0.28209479177387814f;
  b[1] = -0.4886025119029199f * y;
  b[2] = 0.4886025119029199f * z;
  b[3] = -0.4886025119029199f * x;
  b[4] = 1.0925484305920792f * x * y;
  b[5] = -1.0925484305920792f * y * z;
  b[6] = 0.31539156525252005f * (2.f * zz - xx - yy);
  b[7] = -1.0925484305920792f * x * z;
  b[8] = 0.5462742152960396f * (xx - yy);
  b[9] = -0.5900435899266435f * y * (3.f * xx - yy);
  b[10] = 2.890611442640554f * x * y * z;
  b[11] = -0.4570457994644658f * y * (4.f * zz - xx - yy);
  b[12] = 0.3731763325901154f * z * (2.f * zz - 3.f * xx - 3.f * yy);
  b[13] = -0.4570457994644658f * x * (4.f * zz - xx - yy);
  b[14] = 1.445305721320277f * z * (xx - yy);
  b[15] = -0.5900435899266435f * x * (xx - 3.f * yy);
}

template <int NC>
__global__ void __launch_bounds__(kGridThreads)
    grid_render_kernel(const GParams g, const mipnerf_b200_rays rays, float step, int white_bkgd,
                       float* __restrict__ rgb_out, float* __restrict__ dist_out, float* __restrict__ acc_out) {
  const int64_t r = (int64_t)blockIdx.x * kGridThreads + threadIdx.x;
  if (r >= rays.num_rays) return;
  float o[3], d[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) o[a] = __ldg(rays.origins + 3 * r + a), d[a] = __ldg(rays.directions + 3 * r + a);
  const float radius = __ldg(rays.radii + r), near = __ldg(rays.near + r), far = __ldg(rays.far + r);
  float y[16];
  sh_basis(__ldg(rays.viewdirs + 3 * r), __ldg(rays.viewdirs + 3 * r + 1), __ldg(rays.viewdirs + 3 * r + 2), y);

  // the sample lattice, every operation rounded as the contract states
  const float dn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
  const float span = __fsub_rn(far, near);
  const float kf = ceilf(__fdiv_rn(__fmul_rn(span, dn), step));
  const int64_t K = kf >= 1.f ? (int64_t)fminf(kf, 4e18f) : 1;
  const float dt = __fdiv_rn(span, (float)K);
  const float delta = __fmul_rn(dt, dn);

  // clip [0, K) to the samples inside the bounds grown by a margin: t_k increases with k only for dt > 0
  int64_t k0 = 0, k1 = K;
  if (dt > 0.f) {
    float omax = 0.f, dmax = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) omax = fmaxf(omax, fabsf(o[a])), dmax = fmaxf(dmax, fabsf(d[a]));
    const float margin = 1e-5f * (1.f + omax + fmaxf(fabsf(near), fabsf(far)) * dmax + g.bound_mag);
    float t0 = -INFINITY, t1 = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float blo = g.lo[a] - margin, bhi = g.hi[a] + margin;
      if (d[a] != 0.f) {
        const float ta = (blo - o[a]) / d[a], tb = (bhi - o[a]) / d[a];
        t0 = fmaxf(t0, fminf(ta, tb));
        t1 = fminf(t1, fmaxf(ta, tb));
      } else if (!(o[a] >= blo && o[a] <= bhi)) {
        t1 = -INFINITY;  // parallel to the slab and outside it
      }
    }
    if (t1 < t0) {
      k1 = 0;
    } else {
      k0 = first_past(t0, near, dt, 0, K);  // t_k <= t0: outside (t_k == t0 is on the grown box)
      k1 = first_past(t1, near, dt, k0, K);
    }
  }

  const GLevel& l0 = g.lv[0];
  float T = 1.f, acc = 0.f, dist = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
  for (int64_t k = k0; k < k1;) {
    const float t = sample_t(near, dt, k);
    float x[3];
    bool inside = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      x[a] = __fadd_rn(o[a], __fmul_rn(t, d[a]));
      inside = inside && x[a] >= g.lo[a] && x[a] <= g.hi[a];
    }
    if (!inside) {
      ++k;
      continue;
    }
    if (dt > 0.f) {
      int c[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const int i = (int)fminf(fmaxf((x[a] - g.lo[a]) * l0.inv_s[a], 0.f), (float)(l0.n[a] - 2));
        c[a] = i / g.block;
      }
      if (!__ldg(g.occ + ((int64_t)c[2] * g.on[1] + c[1]) * g.on[0] + c[0])) {
        float t_exit = INFINITY;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          if (d[a] == 0.f) continue;
          const int p = d[a] > 0.f ? min((c[a] + 1) * g.block, l0.n[a] - 1) : c[a] * g.block;
          t_exit = fminf(t_exit, (g.lo[a] + (float)p * g.s0[a] - o[a]) / d[a]);
        }
        const int64_t next = first_past(t_exit, near, dt, k, k1);
        k = next > k ? next : k + 1;
        continue;
      }
    }
    float lam = log2f(kSqrt3 * radius * t / g.s0_max);
    lam = fminf(fmaxf(lam, 0.f), (float)(g.num_levels - 1));  // NaN -> 0
    const int la = min((int)lam, g.num_levels - 1);
    const float f = la == g.num_levels - 1 ? 0.f : lam - (float)la;
    int row_a[8], row_b[8];
    float w_a[8], w_b[8];
    float sigma = level_density(g.lv[la], g.lo, x, row_a, w_a);
    if (f > 0.f) sigma = (1.f - f) * sigma + f * level_density(g.lv[la + 1], g.lo, x, row_b, w_b);
    ++k;
    if (!(sigma != 0.f)) continue;
    const float alpha = 1.f - expf(-sigma * delta);
    const float w = T * alpha;
    float raw[3] = {0.f, 0.f, 0.f};
    level_color<NC>(g.lv[la].sh, row_a, w_a, y, f > 0.f ? 1.f - f : 1.f, raw);
    if (f > 0.f) level_color<NC>(g.lv[la + 1].sh, row_b, w_b, y, f, raw);
    const float c0 = g.rgb_scale / (1.f + expf(-raw[0])) - g.rgb_padding;
    const float c1 = g.rgb_scale / (1.f + expf(-raw[1])) - g.rgb_padding;
    const float c2 = g.rgb_scale / (1.f + expf(-raw[2])) - g.rgb_padding;
    cr += w * c0, cg += w * c1, cb += w * c2;
    acc += w;
    dist += w * t;
    T *= 1.f - alpha;
    if (T < kStopTransmittance) break;
  }
  const float bg = white_bkgd ? 1.f - acc : 0.f;
  rgb_out[3 * r] = cr + bg;
  rgb_out[3 * r + 1] = cg + bg;
  rgb_out[3 * r + 2] = cb + bg;
  acc_out[r] = acc;
  dist_out[r] = fminf(fmaxf(dist, near), far);
}

}  // namespace

cudaError_t launch_grid_render(const mipnerf_b200_grid& grid, const mipnerf_b200_rays& rays, float step,
                               int white_bkgd, float* rgb, float* distance, float* acc, cudaStream_t st) {
  if (rays.num_rays == 0) return cudaSuccess;
  GParams g{};
  g.num_levels = grid.num_levels;
  g.nc = (grid.degree + 1) * (grid.degree + 1);
  g.bound_mag = 0.f;
  for (int a = 0; a < 3; ++a) {
    g.lo[a] = grid.lo[a];
    g.hi[a] = grid.hi[a];
    g.bound_mag = fmaxf(g.bound_mag, fmaxf(fabsf(grid.lo[a]), fabsf(grid.hi[a])));
  }
  for (int l = 0; l < grid.num_levels; ++l) {
    const mipnerf_b200_grid_level& s = grid.levels[l];
    GLevel& v = g.lv[l];
    v.cells = reinterpret_cast<const int2*>(s.cells);
    v.sh = s.sh;
    v.n[0] = s.nx, v.n[1] = s.ny, v.n[2] = s.nz;
    for (int a = 0; a < 3; ++a) v.inv_s[a] = (float)(v.n[a] - 1) / (grid.hi[a] - grid.lo[a]);
  }
  g.s0_max = 0.f;
  for (int a = 0; a < 3; ++a) {
    g.s0[a] = (grid.hi[a] - grid.lo[a]) / (float)(g.lv[0].n[a] - 1);
    g.s0_max = fmaxf(g.s0_max, g.s0[a]);
    g.on[a] = (g.lv[0].n[a] - 1 + grid.block - 1) / grid.block;
  }
  g.rgb_scale = 1.f + 2.f * grid.rgb_padding;
  g.rgb_padding = grid.rgb_padding;
  g.occ = grid.occupancy;
  g.block = grid.block;
  const unsigned blocks = (unsigned)((rays.num_rays + kGridThreads - 1) / kGridThreads);
  LaunchScope scope(kKernGridRender, st);
  switch (grid.degree) {
    case 0: grid_render_kernel<1><<<blocks, kGridThreads, 0, st>>>(g, rays, step, white_bkgd, rgb, distance, acc); break;
    case 1: grid_render_kernel<4><<<blocks, kGridThreads, 0, st>>>(g, rays, step, white_bkgd, rgb, distance, acc); break;
    case 2: grid_render_kernel<9><<<blocks, kGridThreads, 0, st>>>(g, rays, step, white_bkgd, rgb, distance, acc); break;
    default: grid_render_kernel<16><<<blocks, kGridThreads, 0, st>>>(g, rays, step, white_bkgd, rgb, distance, acc);
  }
  return cudaGetLastError();
}

}  // namespace mipnerf
