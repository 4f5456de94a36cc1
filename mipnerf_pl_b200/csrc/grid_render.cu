// grid_render.cu — ray marching through a baked grid (mipnerf_b200_grid_render; the grid is built by
// mipnerf_pl_b200/baked.py, which owns the other half of the memory layout read here).
//
// One thread per ray, rays in the caller's (pixel) order, so that neighbouring threads walk neighbouring paths through
// the same cache lines.  Every kernel walks its ray with one of two loops, each written once:
//   * walk_samples, the march over the sample lattice of a step: the render, both passes of its backward, and the
//     visibility scores.  Each caller composites the samples it is handed and keeps its own rule for zero density.
//   * walk_intervals, over the caller's fenceposts: the proposal weights and both passes of their backward.
// Per ray of walk_samples:
//   * K, dt, t_k, delta and the sample positions o + t_k d are computed with explicitly rounded fp32 operations, so a
//     host restatement reproduces them exactly (tests/grid_render_ref.py).
//   * The sample range is first clipped to the bounds grown by a margin far above the rounding of those positions;
//     a sample outside the bounds has density 0, so clipping changes nothing.
//   * Inside, the macro cell of the sample is looked up in the occupancy grid.  An empty cell jumps k to the first
//     sample whose t is past the cell's exit t.  The occupancy builder marks a cell empty only when every level's
//     density is 0 on the cell's lattice points widened by one point of that level, so every skipped sample, and any
//     sample a rounding error away from the cell, interpolates to exactly 0 at every level: skipping is bit-exact.
//   * Density at the level(s) picked by the cone footprint is trilinear over the packed (density, SH row) lattice
//     points (one 8-byte load per corner), read from the dense cells or, in mipnerf_b200_grid_render_bricks, from
//     8^3-point bricks through a brick table.  Colour is evaluated only where the density is non-zero: each kept corner's
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

// Per level the maxima of mipnerf_b200_grid_visibility, indexed by SH row (NULL for a level without kept points).
struct GMaxWeight {
  float* w[MIPNERF_B200_GRID_MAX_LEVELS];
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

// Cell readers: how level_density reads the 8-byte (density bits, SH row) words of one level.  `cells.level(g, l)` is
// level l's reader, and `.cell(lv, i)` (lv = g.lv[l], i the cell's low corner, 0 <= i <= n - 2 per axis) the cell,
// whose `(dx, dy, dz)` is the word of corner i + (dx, dy, dz).  DenseCells reads GLevel::cells, the [nz, ny, nx]
// array.  BrickCells reads the 8^3-point bricks of mipnerf_b200_grid_render_bricks.  Both run the one march below.
struct DenseCells {
  struct Cell {
    const int2* p;
    int64_t sy, sz;
    __device__ __forceinline__ int2 operator()(int dx, int dy, int dz) const { return __ldg(p + dx + dy * sy + dz * sz); }
  };
  struct Level {
    __device__ __forceinline__ Cell cell(const GLevel& l, const int (&i)[3]) const {
      const int64_t base = ((int64_t)i[2] * l.n[1] + i[1]) * l.n[0] + i[0];
      return {l.cells + base, l.n[0], (int64_t)l.n[0] * l.n[1]};
    }
  };
  __device__ __forceinline__ Level level(const GParams&, int) const { return {}; }
};

// Lattice point (i, j, k) is point (i & 7, j & 7, k & 7) of brick (i >> 3, j >> 3, k >> 3); a brick's table entry is
// its id in the pool, or -1 for a brick not stored, whose words all read (+0.0 bits, -1).  Along each axis the cell's
// two corners share a brick unless the low corner is the brick's last point (i & 7 == 7), so 7 of 8 cells per axis
// lie in one brick.  The cell therefore looks up the low corner's brick once and each other corner's only when that
// corner crosses a brick face on an axis where the cell does: a predicated load, not a branch, so the common cell costs
// one table load and a warp whose threads disagree does not diverge.  The kernel takes this by value as a
// __grid_constant__ parameter.
struct BrickCells {
  mipnerf_b200_grid_bricks t;
  struct Cell {
    const int* table;
    const int2* pool;
    int o[3];      // the low corner's local point in its brick
    bool nx[3];    // whether the high corner is in the next brick along the axis
    int64_t bs[3];  // table strides (1, tx, tx * ty)
    int64_t b0;    // the low corner's table entry
    int id0;
    __device__ __forceinline__ int2 operator()(int dx, int dy, int dz) const {
      int id = id0;
      if ((dx && nx[0]) || (dy && nx[1]) || (dz && nx[2]))
        id = __ldg(table + b0 + (dx && nx[0] ? bs[0] : 0) + (dy && nx[1] ? bs[1] : 0) + (dz && nx[2] ? bs[2] : 0));
      const int local = ((((o[2] + dz) & 7) << 3 | ((o[1] + dy) & 7)) << 3) | ((o[0] + dx) & 7);
      return id >= 0 ? __ldg(pool + (int64_t)id * 512 + local) : make_int2(0, -1);
    }
  };
  struct Level {
    const int* table;
    const int2* pool;
    __device__ __forceinline__ Cell cell(const GLevel& l, const int (&i)[3]) const {
      Cell c;
      c.table = table, c.pool = pool;
      const int64_t tx = (l.n[0] + 7) >> 3, ty = (l.n[1] + 7) >> 3;
      c.bs[0] = 1, c.bs[1] = tx, c.bs[2] = tx * ty;
#pragma unroll
      for (int a = 0; a < 3; ++a) c.o[a] = i[a] & 7, c.nx[a] = c.o[a] == 7;
      c.b0 = ((int64_t)(i[2] >> 3) * ty + (i[1] >> 3)) * tx + (i[0] >> 3);
      c.id0 = __ldg(table + c.b0);
      return c;
    }
  };
  __device__ __forceinline__ Level level(const GParams&, int l) const {
    return {t.table[l], reinterpret_cast<const int2*>(t.pool[l])};
  }
};

// Trilinear density of one level at position x: also the corner rows and weights, for the colour.
template <class CellLevel>
__device__ __forceinline__ float level_density(const GLevel& l, const CellLevel cells, const float (&lo)[3],
                                               const float (&x)[3], int (&row)[8], float (&wc)[8]) {
  int i[3];
  float f[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float u = fminf(fmaxf((x[a] - lo[a]) * l.inv_s[a], 0.f), (float)(l.n[a] - 1));
    i[a] = min((int)u, l.n[a] - 2);
    f[a] = u - (float)i[a];
  }
  const auto cell = cells.cell(l, i);
  float sigma = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
    const int2 v = cell(dx, dy, dz);
    wc[c] = (dx ? f[0] : 1.f - f[0]) * (dy ? f[1] : 1.f - f[1]) * (dz ? f[2] : 1.f - f[2]);
    row[c] = v.y;
    sigma += wc[c] * __int_as_float(v.x);
  }
  return sigma;
}

// Row readers: how level_color reads the SH coefficients of one level.  `rows.level(g, l)` is level l's reader, and
// `.row<NC>(r)(k, ch)` coefficient k, channel ch of its SH row r.  F32Rows reads GLevel::sh as stored.  U8Rows reads
// the uint8 rows of mipnerf_b200_grid_render_u8 and dequantizes each coefficient as fl(fl(q * scale) + offset), two
// explicitly rounded fp32 operations (never an FMA), so a u8 render equals the fp32 render of the dequantized rows bit
// for bit.  Both run the one march below: same coefficient order, same accumulation.
struct F32Rows {
  struct Row {
    const float* __restrict__ p;
    __device__ __forceinline__ float operator()(int k, int ch) const { return __ldg(p + 3 * k + ch); }
  };
  struct Level {
    const float* __restrict__ sh;
    template <int NC>
    __device__ __forceinline__ Row row(int r) const { return {sh + (int64_t)r * (NC * 3)}; }
  };
  __device__ __forceinline__ Level level(const GParams& g, int l) const { return {g.lv[l].sh}; }
};

// The kernel takes this by value as a __grid_constant__ parameter: the scale / offset tables are read from the
// parameter space in place, with no copy to a stack frame.
struct U8Rows {
  mipnerf_b200_grid_sh_u8 t;
  struct Row {
    const uint8_t* p;
    const float (*scale)[3];
    const float (*offset)[3];
    __device__ __forceinline__ float operator()(int k, int ch) const {
      return __fadd_rn(__fmul_rn((float)__ldg(p + 3 * k + ch), scale[k][ch]), offset[k][ch]);
    }
  };
  struct Level {
    const uint8_t* rows;
    const float (*scale)[3];
    const float (*offset)[3];
    template <int NC>
    __device__ __forceinline__ Row row(int r) const { return {rows + (int64_t)r * (NC * 3), scale, offset}; }
  };
  __device__ __forceinline__ Level level(const GParams&, int l) const { return {t.rows[l], t.scale[l], t.offset[l]}; }
};

// sum over kept corners of weight * Y . c (raw colour, 3 channels)
template <int NC, class Level>
__device__ __forceinline__ void level_color(const Level sh, const int (&row)[8], const float (&wc)[8],
                                            const float (&y)[16], float scale, float (&raw)[3]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (row[c] < 0) continue;
    const auto p = sh.template row<NC>(row[c]);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      s0 += y[k] * p(k, 0);
      s1 += y[k] * p(k, 1);
      s2 += y[k] * p(k, 2);
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

// One ray's origin, direction, cone radius and |d|, rounded as mipnerf_b200.h states.  Both walks start here; the
// interval walk reads nothing else of the ray (no viewdirs, near or far).
struct Ray {
  float o[3], d[3];
  float radius, dn;
};

__device__ __forceinline__ void load_ray(const mipnerf_b200_rays& rays, int64_t r, Ray& p) {
#pragma unroll
  for (int a = 0; a < 3; ++a) p.o[a] = __ldg(rays.origins + 3 * r + a), p.d[a] = __ldg(rays.directions + 3 * r + a);
  p.radius = __ldg(rays.radii + r);
  p.dn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(p.d[0], p.d[0]), __fmul_rn(p.d[1], p.d[1])),
                              __fmul_rn(p.d[2], p.d[2])));
}

// Position x = o + t d of a ray, each coordinate fl(o + fl(t d)); whether x is inside the bounds.
__device__ __forceinline__ bool ray_point(const GParams& g, const Ray& p, float t, float (&x)[3]) {
  bool inside = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    x[a] = __fadd_rn(p.o[a], __fmul_rn(t, p.d[a]));
    inside = inside && x[a] >= g.lo[a] && x[a] <= g.hi[a];
  }
  return inside;
}

// One ray's sample lattice, clipped to the samples inside the bounds grown by a margin.
struct RayMarch : Ray {
  float near, far;
  float dt, delta;
  int64_t k0, k1;
};

__device__ __forceinline__ void ray_setup(const GParams& g, const mipnerf_b200_rays& rays, int64_t r, float step,
                                          RayMarch& m, float (&y)[16]) {
  load_ray(rays, r, m);
  m.near = __ldg(rays.near + r), m.far = __ldg(rays.far + r);
  sh_basis(__ldg(rays.viewdirs + 3 * r), __ldg(rays.viewdirs + 3 * r + 1), __ldg(rays.viewdirs + 3 * r + 2), y);
  const float(&o)[3] = m.o;
  const float(&d)[3] = m.d;
  const float near = m.near, far = m.far, dn = m.dn;

  // the sample lattice, every operation rounded as the contract states
  const float span = __fsub_rn(far, near);
  const float kf = ceilf(__fdiv_rn(__fmul_rn(span, dn), step));
  const int64_t K = kf >= 1.f ? (int64_t)fminf(kf, 4e18f) : 1;
  const float dt = __fdiv_rn(span, (float)K);
  m.dt = dt;
  m.delta = __fmul_rn(dt, dn);

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
  m.k0 = k0, m.k1 = k1;
}

// Whether the macro cell of an inside position x is occupied; c is the cell.
__device__ __forceinline__ bool occupied(const GParams& g, const float (&x)[3], int (&c)[3]) {
  const GLevel& l0 = g.lv[0];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int i = (int)fminf(fmaxf((x[a] - g.lo[a]) * l0.inv_s[a], 0.f), (float)(l0.n[a] - 2));
    c[a] = i / g.block;
  }
  return __ldg(g.occ + ((int64_t)c[2] * g.on[1] + c[1]) * g.on[0] + c[0]);
}

// For dt > 0: if x lies in an empty macro cell, move k to the first sample past the cell's exit t (at least k + 1) and
// return true.
__device__ __forceinline__ bool skip_empty(const GParams& g, const RayMarch& m, const float (&x)[3], int64_t& k) {
  const GLevel& l0 = g.lv[0];
  int c[3];
  if (occupied(g, x, c)) return false;
  float t_exit = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (m.d[a] == 0.f) continue;
    const int p = m.d[a] > 0.f ? min((c[a] + 1) * g.block, l0.n[a] - 1) : c[a] * g.block;
    t_exit = fminf(t_exit, (g.lo[a] + (float)p * g.s0[a] - m.o[a]) / m.d[a]);
  }
  const int64_t next = first_past(t_exit, m.near, m.dt, k, m.k1);
  k = next > k ? next : k + 1;
  return true;
}

// The level(s) the cone footprint picks at a sample, with both levels' corner rows and weights.
struct Blend {
  int la;
  float f;  // weight of level la + 1; level la has 1 - f (1 when f == 0, and level la + 1 is not read)
  int row_a[8], row_b[8];
  float w_a[8], w_b[8];

  // visit(l, row, wc, lw) for each level the blend reads: its corner rows and weights and its level weight.
  template <class Visit>
  __device__ __forceinline__ void levels(Visit&& visit) const {
    visit(la, row_a, w_a, f > 0.f ? 1.f - f : 1.f);
    if (f > 0.f) visit(la + 1, row_b, w_b, f);
  }
};

template <class Cells>
__device__ __forceinline__ float blend_density(const GParams& g, const Cells& cells, float radius, float t,
                                               const float (&x)[3], Blend& b) {
  float lam = log2f(kSqrt3 * radius * t / g.s0_max);
  lam = fminf(fmaxf(lam, 0.f), (float)(g.num_levels - 1));  // NaN -> 0
  b.la = min((int)lam, g.num_levels - 1);
  b.f = b.la == g.num_levels - 1 ? 0.f : lam - (float)b.la;
  float sigma = level_density(g.lv[b.la], cells.level(g, b.la), g.lo, x, b.row_a, b.w_a);
  if (b.f > 0.f)
    sigma = (1.f - b.f) * sigma +
            b.f * level_density(g.lv[b.la + 1], cells.level(g, b.la + 1), g.lo, x, b.row_b, b.w_b);
  return sigma;
}

// The blended raw colour Y . c of a sample.
template <int NC, class Rows>
__device__ __forceinline__ void blend_raw(const GParams& g, const Rows& rows, const Blend& b, const float (&y)[16],
                                          float (&raw)[3]) {
  raw[0] = raw[1] = raw[2] = 0.f;
  b.levels([&](int l, const int (&row)[8], const float (&wc)[8], float lw) {
    level_color<NC>(rows.level(g, l), row, wc, y, lw, raw);
  });
}

// The samples of a ray's march whose density is looked up, front to back: inside the bounds and, for dt > 0, not in
// an empty macro cell.  keep(sigma, b) is the caller's rule for which of them it uses (its rule for zero density), and
// visit(t, sigma, b) is called for those, with the sample's t, blended density and level blend; the walk goes on while
// visit returns true.  The rule is a separate argument, and visit's result means "go on" rather than "stop", because
// in that loop shape no kernel spills: with the rule inside visit or a "stop" result, ptxas (CUDA 12.9) gives the
// degree-2 uint8 brick render a 16-byte stack frame at its 96 registers.
template <class Cells, class Keep, class Visit>
__device__ __forceinline__ void walk_samples(const GParams& g, const Cells& cells, const RayMarch& m, Keep&& keep,
                                             Visit&& visit) {
  for (int64_t k = m.k0; k < m.k1;) {
    const float t = sample_t(m.near, m.dt, k);
    float x[3];
    if (!ray_point(g, m, t, x)) {
      ++k;
      continue;
    }
    if (m.dt > 0.f && skip_empty(g, m, x, k)) continue;
    Blend b;
    const float sigma = blend_density(g, cells, m.radius, t, x, b);
    ++k;
    if (!keep(sigma, b)) continue;
    if (!visit(t, sigma, b)) break;
  }
}

// Front-to-back compositing state: transmittance and the running sums of the outputs.
struct Composite {
  float T = 1.f, acc = 0.f, dist = 0.f, c[3] = {0.f, 0.f, 0.f};
};

__device__ __forceinline__ void composite(Composite& s, float alpha, const float (&c)[3], float t) {
  const float w = s.T * alpha;
  s.c[0] += w * c[0], s.c[1] += w * c[1], s.c[2] += w * c[2];
  s.acc += w;
  s.dist += w * t;
  s.T *= 1.f - alpha;
}

// The forward march of one ray: every sample with non-zero density composited, up to the one that leaves T < 1e-4.
template <int NC, class Rows, class Cells>
__device__ __forceinline__ void march(const GParams& g, const Rows& rows, const Cells& cells, const RayMarch& m,
                                      const float (&y)[16], Composite& s) {
  const auto nonzero = [](float sigma, const Blend&) { return sigma != 0.f; };
  walk_samples(g, cells, m, nonzero, [&](float t, float sigma, const Blend& b) {
    const float alpha = 1.f - expf(-sigma * m.delta);
    float raw[3], c[3];
    blend_raw<NC>(g, rows, b, y, raw);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) c[ch] = g.rgb_scale / (1.f + expf(-raw[ch])) - g.rgb_padding;
    composite(s, alpha, c, t);
    return !(s.T < kStopTransmittance);
  });
}

template <int NC, class Rows, class Cells>
__global__ void __launch_bounds__(kGridThreads)
    grid_render_kernel(const GParams g, const mipnerf_b200_rays rays, float step, int white_bkgd,
                       float* __restrict__ rgb_out, float* __restrict__ dist_out, float* __restrict__ acc_out,
                       const __grid_constant__ Rows rows, const __grid_constant__ Cells cells) {
  const int64_t r = (int64_t)blockIdx.x * kGridThreads + threadIdx.x;
  if (r >= rays.num_rays) return;
  RayMarch m;
  float y[16];
  ray_setup(g, rays, r, step, m, y);
  Composite s;
  march<NC>(g, rows, cells, m, y, s);
  const float bg = white_bkgd ? 1.f - s.acc : 0.f;
  rgb_out[3 * r] = s.c[0] + bg;
  rgb_out[3 * r + 1] = s.c[1] + bg;
  rgb_out[3 * r + 2] = s.c[2] + bg;
  acc_out[r] = s.acc;
  dist_out[r] = fminf(fmaxf(s.dist, m.near), m.far);
}

// Add one level's share of a sample's gradients into the kept corners: density with weight lw * wc, each SH
// coefficient with lw * wc * Y_k (only when the colour has a gradient).
template <int NC>
__device__ __forceinline__ void level_scatter(float* __restrict__ gd, float* __restrict__ gsh, const int (&row)[8],
                                              const float (&wc)[8], float lw, const float (&y)[16], float d_sigma,
                                              const float (&d_raw)[3], bool color) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (row[c] < 0) continue;
    const float w = lw * wc[c];
    atomicAdd(gd + row[c], w * d_sigma);
    if (!color) continue;
    float* p = gsh + (int64_t)row[c] * (NC * 3);
    const float a0 = w * d_raw[0], a1 = w * d_raw[1], a2 = w * d_raw[2];
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      atomicAdd(p + 3 * k, y[k] * a0);
      atomicAdd(p + 3 * k + 1, y[k] * a1);
      atomicAdd(p + 3 * k + 2, y[k] * a2);
    }
  }
}

// Whether a level the blend reads has a kept corner.
__device__ __forceinline__ bool any_kept(const Blend& b) {
  bool any = false;
  b.levels([&](int, const int (&row)[8], const float (&)[8], float) {
#pragma unroll
    for (int c = 0; c < 8; ++c) any = any || row[c] >= 0;
  });
  return any;
}

// The gradient of grid_render_kernel's outputs, one thread per ray.  Pass 1 is the forward march (its totals: the
// foreground rgb, acc and the unclamped distance).  Pass 2 walks with march's walk_samples over the same cells, so it
// is handed the same samples; it also keeps a zero density with a kept corner, but composites only the samples march
// composites, with composite, and stops where march stops.  So the prefix sums it forms equal the totals bit for bit
// at the last composited sample.  With
// e_k = g_rgb . c_k + g_acc' + g_dist t_k (g_acc' = g_acc - sum g_rgb under a white background) and w_k = T_k alpha_k,
// dL/dsigma_k = delta (T_{k+1} e_k - sum_{j > k} w_j e_j), the suffix being total - prefix, and dL/draw_k = w_k g_rgb
// (1 + 2 rgb_padding) s (1 - s) for s the sigmoid of the raw colour.
template <int NC>
__global__ void __launch_bounds__(kGridThreads)
    grid_render_backward_kernel(const GParams g, const mipnerf_b200_rays rays, float step, int white_bkgd,
                                const float* __restrict__ d_rgb, const float* __restrict__ d_dist,
                                const float* __restrict__ d_acc,
                                const __grid_constant__ mipnerf_b200_grid_grads grads) {
  const int64_t r = (int64_t)blockIdx.x * kGridThreads + threadIdx.x;
  if (r >= rays.num_rays) return;
  float g_rgb[3] = {0.f, 0.f, 0.f};
  if (d_rgb) g_rgb[0] = d_rgb[3 * r], g_rgb[1] = d_rgb[3 * r + 1], g_rgb[2] = d_rgb[3 * r + 2];
  float g_acc = d_acc ? d_acc[r] : 0.f, g_dist = d_dist ? d_dist[r] : 0.f;
  if (white_bkgd) g_acc -= g_rgb[0] + g_rgb[1] + g_rgb[2];
  if (g_rgb[0] == 0.f && g_rgb[1] == 0.f && g_rgb[2] == 0.f && g_acc == 0.f && g_dist == 0.f) return;
  RayMarch m;
  float y[16];
  ray_setup(g, rays, r, step, m, y);
  Composite total;
  march<NC>(g, F32Rows{}, DenseCells{}, m, y, total);
  if (!(total.dist >= m.near && total.dist <= m.far)) g_dist = 0.f;  // the clamp passes the gradient inside, inclusive

  Composite s;
  // a zero density still has a gradient; it reaches parameters only through kept corners
  const auto has_gradient = [](float sigma, const Blend& b) { return sigma != 0.f || any_kept(b); };
  walk_samples(g, DenseCells{}, m, has_gradient, [&](float t, float sigma, const Blend& b) {
    const bool zero = !(sigma != 0.f);
    const float alpha = 1.f - expf(-sigma * m.delta);
    float raw[3], c[3], sg[3];
    blend_raw<NC>(g, F32Rows{}, b, y, raw);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      sg[ch] = 1.f / (1.f + expf(-raw[ch]));
      c[ch] = g.rgb_scale / (1.f + expf(-raw[ch])) - g.rgb_padding;
    }
    const float w = s.T * alpha;
    if (!zero) composite(s, alpha, c, t);  // s.T is now T_{k+1}, the prefix sums include this sample
    const float suffix = g_rgb[0] * (total.c[0] - s.c[0]) + g_rgb[1] * (total.c[1] - s.c[1]) +
                         g_rgb[2] * (total.c[2] - s.c[2]) + g_acc * (total.acc - s.acc) +
                         g_dist * (total.dist - s.dist);
    const float e = g_rgb[0] * c[0] + g_rgb[1] * c[1] + g_rgb[2] * c[2] + g_acc + g_dist * t;
    const float d_sigma = m.delta * (s.T * e - suffix);
    float d_raw[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) d_raw[ch] = w * g_rgb[ch] * g.rgb_scale * sg[ch] * (1.f - sg[ch]);
    const bool color = !zero;  // w == 0 at a zero density
    b.levels([&](int l, const int (&row)[8], const float (&wc)[8], float lw) {
      level_scatter<NC>(grads.density[l], grads.sh[l], row, wc, lw, y, d_sigma, d_raw, color);
    });
    return !(s.T < kStopTransmittance);
  });
}

// Raise one level's kept corners to their scores at a composited sample of blending weight w: corner c's score is
// w * (lw * wc[c]), w times the coefficient level_color gives the corner's colour.  The maximum is an integer atomicMax
// on the float's bits, which orders non-negative floats as the floats; a negative score (from a negative density)
// never raises an entry the caller started at 0.  The plain load in front skips the atomic when the entry already
// holds at least the score: entries only grow, so a stale read costs one unneeded atomic and never loses a maximum.
__device__ __forceinline__ void level_visibility(float* __restrict__ max_weight, const int (&row)[8],
                                                 const float (&wc)[8], float lw, float w) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (row[c] < 0) continue;
    const int s = __float_as_int(w * (lw * wc[c]));
    int* p = reinterpret_cast<int*>(max_weight) + row[c];
    if (s > *p) atomicMax(p, s);
  }
}

// Per kept corner, the largest score over these rays (mipnerf_b200_grid_visibility), one thread per ray.  It walks with
// march's walk_samples and zero-density rule, for density only: it is handed the forward's samples, level blends and
// trilinear weights, forms w_k = T_k alpha_k with composite's arithmetic on T, and stops after the sample that leaves
// T < 1e-4; no colour is evaluated.  A maximum does not depend on the order of its updates, so the result is bit for
// bit the same across runs, across any split of the rays into calls, and under any permutation of the rays.
// With BrickCells (mipnerf_b200_grid_visibility_bricks) every corner reads the word the dense cells hold, so the scores
// equal the dense kernel's on the densified grid bit for bit.
template <class Cells>
__global__ void __launch_bounds__(kGridThreads)
    grid_visibility_kernel(const GParams g, const mipnerf_b200_rays rays, float step,
                           const __grid_constant__ GMaxWeight max_weight, const __grid_constant__ Cells cells) {
  const int64_t r = (int64_t)blockIdx.x * kGridThreads + threadIdx.x;
  if (r >= rays.num_rays) return;
  RayMarch m;
  float y[16];
  ray_setup(g, rays, r, step, m, y);
  float T = 1.f;
  const auto nonzero = [](float sigma, const Blend&) { return sigma != 0.f; };
  walk_samples(g, cells, m, nonzero, [&](float, float sigma, const Blend& b) {
    const float alpha = 1.f - expf(-sigma * m.delta);
    const float w = T * alpha;
    b.levels([&](int l, const int (&row)[8], const float (&wc)[8], float lw) {
      level_visibility(max_weight.w[l], row, wc, lw, w);
    });
    T *= 1.f - alpha;
    return !(T < kStopTransmittance);
  });
}

// Interval [t0, t1] of a ray: its delta, and the density at its midpoint under the level blend.  A midpoint outside
// the bounds or in an empty macro cell is not looked up (density 0, `looked_up` false, `b` unset).
template <class Cells>
__device__ __forceinline__ float proposal_density(const GParams& g, const Cells& cells, const Ray& p, float t0,
                                                  float t1, float& delta, Blend& b, bool& looked_up) {
  const float tm = __fmul_rn(__fadd_rn(t0, t1), 0.5f);
  delta = __fmul_rn(__fsub_rn(t1, t0), p.dn);
  float x[3];
  const bool inside = ray_point(g, p, tm, x);
  float sigma = 0.f;
  int c[3];
  looked_up = false;
  if (inside && occupied(g, x, c)) {
    looked_up = true;
    sigma = blend_density(g, cells, p.radius, tm, x, b);
  }
  return sigma;
}

// The n intervals of a ray between its fenceposts t[0..n], front to back, with volumetric_rendering's weights and no
// stop: s_i = fl(sigma_i delta_i) from proposal_density, w_i = fl(fl(1 - e^{-s_i}) e^{-S_i}) and S_{i+1} = fl(S_i +
// s_i), S_0 = 0, every rounding as mipnerf_b200.h states.  visit(i, w_i, S_{i+1}, delta_i, looked_up, b) for each.
template <class Cells, class Visit>
__device__ __forceinline__ void walk_intervals(const GParams& g, const Cells& cells, const Ray& p, const float* t,
                                               int n, Visit&& visit) {
  float S = 0.f;
  float t0 = __ldg(t);
  for (int i = 0; i < n; ++i) {
    const float t1 = __ldg(t + i + 1);
    float delta;
    Blend b;
    bool looked_up;
    const float s = __fmul_rn(proposal_density(g, cells, p, t0, t1, delta, b, looked_up), delta);
    t0 = t1;
    const float w = __fmul_rn(__fsub_rn(1.f, expf(-s)), expf(-S));
    S = __fadd_rn(S, s);
    visit(i, w, S, delta, looked_up, b);
  }
}

// Proposal weights of the caller's intervals (mipnerf_b200_grid_proposal), one thread per ray: walk_intervals' w_i.
// Interval i is sampled at its midpoint with blend_density.  A midpoint in an empty macro cell has density exactly 0
// at every level (the occupancy rule skip_empty relies on), so its lookup is skipped and s_i = 0 exactly: the result
// equals the all-occupied grid's bit for bit.  No SH row is read.
template <class Cells>
__global__ void __launch_bounds__(kGridThreads)
    grid_proposal_kernel(const GParams g, const mipnerf_b200_rays rays, const float* __restrict__ t_samples,
                         int num_samples, float* __restrict__ weights, const __grid_constant__ Cells cells) {
  const int64_t r = (int64_t)blockIdx.x * kGridThreads + threadIdx.x;
  if (r >= rays.num_rays) return;
  Ray p;
  load_ray(rays, r, p);
  float* out = weights + r * num_samples;
  walk_intervals(g, cells, p, t_samples + r * (num_samples + 1), num_samples,
                 [&](int i, float w, float, float, bool, const Blend&) { out[i] = w; });
}

// The gradient of grid_proposal_kernel's weights with respect to the densities (mipnerf_b200_grid_proposal_backward),
// dense fp32 cells, one thread per ray.  With g_i = d_weights[i], s_i = sigma_i delta_i and S_i = sum_{j<i} s_j, w_i =
// e^{-S_i} - e^{-S_{i+1}}, so dL/ds_k = g_k e^{-S_{k+1}} - sum_{i>k} g_i w_i and dL/dsigma_k = delta_k dL/ds_k.  Both
// passes are the forward's walk_intervals, so they are handed the forward's w_i.  Pass 1 sums g_i w_i; pass 2 sums
// them again in the same order, so its prefix sum reaches the total bit for bit, and takes the suffix as total -
// prefix, as grid_render_backward_kernel does.  An interval the forward does not look up (midpoint outside the bounds
// or in an empty macro cell) gets no gradient; the others scatter through the level blend and the trilinear weights
// into the kept corners (level_scatter, density only).
__global__ void __launch_bounds__(kGridThreads)
    grid_proposal_backward_kernel(const GParams g, const mipnerf_b200_rays rays, const float* __restrict__ t_samples,
                                  int num_samples, const float* __restrict__ d_weights,
                                  const __grid_constant__ mipnerf_b200_grid_grads grads) {
  const int64_t r = (int64_t)blockIdx.x * kGridThreads + threadIdx.x;
  if (r >= rays.num_rays) return;
  Ray p;
  load_ray(rays, r, p);
  const float* t = t_samples + r * (num_samples + 1);
  const float* gw = d_weights + r * num_samples;
  float total = 0.f;
  walk_intervals(g, DenseCells{}, p, t, num_samples, [&](int i, float w, float, float, bool, const Blend&) {
    total = __fmaf_rn(__ldg(gw + i), w, total);
  });
  const float y[16] = {};
  const float d_raw[3] = {};
  float prefix = 0.f;
  walk_intervals(g, DenseCells{}, p, t, num_samples,
                 [&](int i, float w, float S, float delta, bool looked_up, const Blend& b) {
                   const float gi = __ldg(gw + i);
                   prefix = __fmaf_rn(gi, w, prefix);
                   if (!looked_up) return;
                   const float d_sigma = delta * (gi * expf(-S) - (total - prefix));
                   if (d_sigma == 0.f) return;
                   b.levels([&](int l, const int (&row)[8], const float (&wc)[8], float lw) {
                     level_scatter<1>(grads.density[l], nullptr, row, wc, lw, y, d_sigma, d_raw, false);
                   });
                 });
}

GParams make_params(const mipnerf_b200_grid& grid) {
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
  return g;
}

unsigned grid_blocks(int64_t num_rays) { return (unsigned)((num_rays + kGridThreads - 1) / kGridThreads); }

// The prologue every launcher below shares: nothing to launch for no rays; otherwise launch(g, blocks) with `grid`'s
// kernel parameters and the grid size of num_rays, timed under profiler id `id`.  Returns the launch's error.
template <class Launch>
cudaError_t launch_rays(const mipnerf_b200_grid& grid, int64_t num_rays, int id, cudaStream_t st, Launch&& launch) {
  if (num_rays == 0) return cudaSuccess;
  const GParams g = make_params(grid);
  LaunchScope scope(id, st);
  launch(g, grid_blocks(num_rays));
  return cudaGetLastError();
}

// f(cells) with the cell reader of the nullable `bricks`: BrickCells over them, or DenseCells for levels[l].cells.
template <class F>
void with_cells(const mipnerf_b200_grid_bricks* bricks, F&& f) {
  if (bricks) return f(BrickCells{*bricks});
  f(DenseCells{});
}

}  // namespace

cudaError_t launch_grid_render(const mipnerf_b200_grid& grid, const mipnerf_b200_grid_bricks* bricks,
                               const mipnerf_b200_grid_sh_u8* sh, const mipnerf_b200_rays& rays, float step,
                               int white_bkgd, float* rgb, float* distance, float* acc, int id, cudaStream_t st) {
  return launch_rays(grid, rays.num_rays, id, st, [&](const GParams& g, unsigned blocks) {
    // the rows: the fp32 levels[l].sh, or the uint8 rows given
    const auto launch = [&](const auto& rows, const auto& cells) {
      using Rows = std::decay_t<decltype(rows)>;
      using Cells = std::decay_t<decltype(cells)>;
      with_sh_coeffs(grid.degree, [&](auto nc) {
        grid_render_kernel<decltype(nc)::value, Rows, Cells><<<blocks, kGridThreads, 0, st>>>(
            g, rays, step, white_bkgd, rgb, distance, acc, rows, cells);
      });
    };
    with_cells(bricks, [&](const auto& cells) {
      if (sh) launch(U8Rows{*sh}, cells);
      else launch(F32Rows{}, cells);
    });
  });
}

cudaError_t launch_grid_render_backward(const mipnerf_b200_grid& grid, const mipnerf_b200_rays& rays, float step,
                                        int white_bkgd, const float* d_rgb, const float* d_distance,
                                        const float* d_acc, const mipnerf_b200_grid_grads& grads, cudaStream_t st) {
  if (!d_rgb && !d_distance && !d_acc) return cudaSuccess;
  return launch_rays(grid, rays.num_rays, kKernGridRenderBackward, st, [&](const GParams& g, unsigned blocks) {
    with_sh_coeffs(grid.degree, [&](auto nc) {
      grid_render_backward_kernel<decltype(nc)::value><<<blocks, kGridThreads, 0, st>>>(
          g, rays, step, white_bkgd, d_rgb, d_distance, d_acc, grads);
    });
  });
}

cudaError_t launch_grid_visibility(const mipnerf_b200_grid& grid, const mipnerf_b200_grid_bricks* bricks,
                                   const mipnerf_b200_rays& rays, float step, float* const* max_weight, int id,
                                   cudaStream_t st) {
  return launch_rays(grid, rays.num_rays, id, st, [&](const GParams& g, unsigned blocks) {
    GMaxWeight mw{};
    for (int l = 0; l < grid.num_levels; ++l) mw.w[l] = max_weight[l];
    with_cells(bricks, [&](const auto& cells) {
      grid_visibility_kernel<std::decay_t<decltype(cells)>><<<blocks, kGridThreads, 0, st>>>(g, rays, step, mw, cells);
    });
  });
}

cudaError_t launch_grid_proposal(const mipnerf_b200_grid& grid, const mipnerf_b200_grid_bricks* bricks,
                                 const mipnerf_b200_rays& rays, const float* t_samples, int num_samples,
                                 float* weights, cudaStream_t st) {
  return launch_rays(grid, rays.num_rays, kKernGridProposal, st, [&](const GParams& g, unsigned blocks) {
    with_cells(bricks, [&](const auto& cells) {
      grid_proposal_kernel<std::decay_t<decltype(cells)>><<<blocks, kGridThreads, 0, st>>>(
          g, rays, t_samples, num_samples, weights, cells);
    });
  });
}

cudaError_t launch_grid_proposal_backward(const mipnerf_b200_grid& grid, const mipnerf_b200_rays& rays,
                                          const float* t_samples, int num_samples, const float* d_weights,
                                          const mipnerf_b200_grid_grads& grads, cudaStream_t st) {
  return launch_rays(grid, rays.num_rays, kKernGridProposalBackward, st, [&](const GParams& g, unsigned blocks) {
    grid_proposal_backward_kernel<<<blocks, kGridThreads, 0, st>>>(g, rays, t_samples, num_samples, d_weights, grads);
  });
}

}  // namespace mipnerf
