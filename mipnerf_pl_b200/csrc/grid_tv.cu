// grid_tv.cu — the total-variation prior of a baked grid (mipnerf_b200_grid_tv; the definition is in
// include/mipnerf_b200.h and mipnerf_pl_b200/baked.py, BakedGrid.total_variation).
//
// One thread per kept point p (SH row r of its level), rows in order.  The thread reads p's lattice position, then the
// 8-byte (density bits, SH row) words of the points its terms and gradient depend on: its 3 forward neighbours
// p + e_a, and for the gradient its 3 backward neighbours b_a = p - e_a and each b_a's two other forward neighbours
// b_a + e_c (c != a), whose differences enter b_a's terms.  It forms p's own terms, and as the derivative of the term
// sums with respect to p's parameters the fixed-order sum of the derivative of p's own term and of each kept b_a's
// term.  Every gradient entry is written by the one thread that formed it: no atomics, bit-reproducible.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/mipnerf_b200.h"
#include "kernels.h"
#include "profile.h"

namespace mipnerf {
namespace {

constexpr int kTvThreads = 128;

struct TvLevel {
  const int2* cells;
  const float* sh;
  const int64_t* pos;  // lattice position of SH row r
  int64_t m;           // rows this launch covers (0: none)
  float* tv_d;
  float* tv_sh;
  float* g_d;
  float* g_sh;
  int n[3];
  int64_t block0;  // the level's first block
};

struct TvParams {
  TvLevel lv[MIPNERF_B200_GRID_MAX_LEVELS];
  int num_levels;
  float eps;
  const float* weights;  // device [2]: density, SH
};

// A lattice point as the terms read it: its SH row (-1 when dropped or outside the lattice) and its density (0 when
// dropped or outside).
struct Nb {
  int row;
  float sigma;
};

__device__ __forceinline__ Nb read_point(const int2* cells, int64_t q, bool inside) {
  Nb b{-1, 0.f};
  if (inside) {
    const int2 w = __ldg(cells + q);
    if (w.y >= 0) b.row = w.y, b.sigma = __int_as_float(w.x);
  }
  return b;
}

template <int NC>
__global__ void __launch_bounds__(kTvThreads) grid_tv_kernel(const __grid_constant__ TvParams P) {
  int l = 0;
  while (l + 1 < P.num_levels && (int64_t)blockIdx.x >= P.lv[l + 1].block0) ++l;
  const TvLevel& L = P.lv[l];
  const int64_t r = ((int64_t)blockIdx.x - L.block0) * kTvThreads + threadIdx.x;
  if (r >= L.m) return;
  constexpr int R = 3 * NC;  // floats per SH row
  const int64_t p = __ldg(L.pos + r);
  const int64_t s[3] = {1, L.n[0], (int64_t)L.n[0] * L.n[1]};
  const int i[3] = {(int)(p % L.n[0]), (int)((p / L.n[0]) % L.n[1]), (int)(p / s[2])};
  const float sp = __int_as_float(__ldg(L.cells + p).x);
  const bool grad_d = L.g_d != nullptr, grad_sh = L.g_sh != nullptr;
  bool fwd[3];  // p + e_a inside the lattice
  Nb f[3], b[3], d[3][3];  // forward, backward, d[a][c] = b_a + e_c (c != a)
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    fwd[a] = i[a] + 1 < L.n[a];
    f[a] = read_point(L.cells, p + s[a], fwd[a]);
  }
  if (grad_d || grad_sh) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      b[a] = read_point(L.cells, p - s[a], i[a] > 0);
#pragma unroll
      for (int c = 0; c < 3; ++c)
        if (c != a) d[a][c] = read_point(L.cells, p - s[a] + s[c], b[a].row >= 0 && fwd[c]);
    }
  }
  const float eps = P.eps;

  // density: a dropped neighbour inside the lattice reads 0, one outside gives a zero difference
  {
    float D[3], q = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      D[a] = fwd[a] ? f[a].sigma - sp : 0.f;
      q += D[a] * D[a];
    }
    const float T = sqrtf(eps + q);
    if (L.tv_d) L.tv_d[r] = T;
    if (grad_d) {
      float g = -((D[0] + D[1] + D[2]) / T);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (b[a].row < 0) continue;
        float qb = 0.f, da = 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float e = c == a ? sp - b[a].sigma : fwd[c] ? d[a][c].sigma - b[a].sigma : 0.f;
          if (c == a) da = e;
          qb += e * e;
        }
        g += da / sqrtf(eps + qb);
      }
      L.g_d[r] = __ldg(P.weights) * g;
    }
  }

  // SH: a difference to a dropped neighbour, or across the lattice's edge, is 0
  if (!L.tv_sh && !grad_sh) return;
  const float* rp = L.sh + r * R;
  const float w_sh = grad_sh ? __ldg(P.weights + 1) : 0.f;
  float term = 0.f;
#pragma unroll 3
  for (int j = 0; j < R; ++j) {
    const float cp = __ldg(rp + j);
    float D[3], q = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      D[a] = f[a].row >= 0 ? __ldg(L.sh + (int64_t)f[a].row * R + j) - cp : 0.f;
      q += D[a] * D[a];
    }
    const float T = sqrtf(eps + q);
    term += T;
    if (!grad_sh) continue;
    float g = -((D[0] + D[1] + D[2]) / T);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (b[a].row < 0) continue;
      const float cb = __ldg(L.sh + (int64_t)b[a].row * R + j);
      float qb = 0.f, da = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float e = c == a ? cp - cb : d[a][c].row >= 0 ? __ldg(L.sh + (int64_t)d[a][c].row * R + j) - cb : 0.f;
        if (c == a) da = e;
        qb += e * e;
      }
      g += da / sqrtf(eps + qb);
    }
    L.g_sh[r * R + j] = w_sh * g;
  }
  if (L.tv_sh) L.tv_sh[r] = term;
}

}  // namespace

cudaError_t launch_grid_tv(const mipnerf_b200_grid& grid, const int64_t* const* points, const int64_t* num_points,
                           float eps, float* const* tv_density, float* const* tv_sh, const float* weights,
                           const mipnerf_b200_grid_grads* grads, cudaStream_t st) {
  TvParams P{};
  P.num_levels = grid.num_levels;
  P.eps = eps;
  P.weights = weights;
  int64_t blocks = 0;
  for (int l = 0; l < grid.num_levels; ++l) {
    const mipnerf_b200_grid_level& s = grid.levels[l];
    TvLevel& v = P.lv[l];
    v.cells = reinterpret_cast<const int2*>(s.cells);
    v.sh = s.sh;
    v.pos = points[l];
    v.n[0] = s.nx, v.n[1] = s.ny, v.n[2] = s.nz;
    v.tv_d = tv_density ? tv_density[l] : nullptr;
    v.tv_sh = tv_sh ? tv_sh[l] : nullptr;
    v.g_d = grads ? grads->density[l] : nullptr;
    v.g_sh = grads ? grads->sh[l] : nullptr;
    v.m = v.tv_d || v.tv_sh || v.g_d || v.g_sh ? num_points[l] : 0;  // a level with no output launches no thread
    v.block0 = blocks;
    blocks += (v.m + kTvThreads - 1) / kTvThreads;
  }
  if (blocks == 0) return cudaSuccess;
  LaunchScope scope(kKernGridTv, st);
  with_sh_coeffs(grid.degree,
                 [&](auto nc) { grid_tv_kernel<decltype(nc)::value><<<(unsigned)blocks, kTvThreads, 0, st>>>(P); });
  return cudaGetLastError();
}

}  // namespace mipnerf
