// isosurface.cu — marching tetrahedra over a scalar grid (mipnerf_b200_isosurface_count / _emit), and the vertex
// normals of the emitted mesh from the grid's gradient (mipnerf_b200_isosurface_normals).
//
// Lattice point (i, j, k) of a grid [nz, ny, nx] (x fastest) sits at lo + idx * step per axis.  Each cell is split into
// the 6 Kuhn tetrahedra v0 -> v0 + e_a -> v0 + e_a + e_b -> v0 + (1,1,1), one per axis permutation (a, b, c), so that
// every tetrahedron edge is a lattice edge from a point in one of 7 positive directions (x, y, z, x+y, x+z, y+z,
// x+y+z).  A point owns those 7 edges.  A value > iso is inside (NaN is outside); an edge with exactly one inside end
// carries one vertex at p_a + t (p_b - p_a), t = (iso - v_a) / (v_b - v_a), a the owner (t = 1/2 when that is NaN).
// Vertex ids are an exclusive scan over (point in x-fastest order, direction); faces an exclusive scan over (cell,
// tetrahedron, triangle).  Both scans run over fixed tiles of kIsoTile points and a fixed-order reduction, so the
// output is bit-reproducible; every float operation is an explicitly rounded one (no contraction), so a numpy
// implementation of the same rules reproduces the vertices bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "profile.h"

namespace mipnerf {
namespace {

constexpr int kIsoThreads = 256;
constexpr int kIsoPer = 8;  // consecutive points per thread
constexpr int kIsoTile = kIsoThreads * kIsoPer;
constexpr int kScanThreads = 1024;

// direction index of a corner offset (bit 0 = x, 1 = y, 2 = z); -1 for the zero offset
__constant__ int8_t c_dir_of_bits[8] = {-1, 0, 1, 3, 2, 4, 5, 6};
__constant__ int8_t c_bits_of_dir[7] = {1, 2, 4, 3, 5, 6, 7};
// the Kuhn tetrahedra as corner offsets, permutations (x,y,z) (x,z,y) (y,x,z) (y,z,x) (z,x,y) (z,y,x); the odd
// permutations have negative orientation
__constant__ int8_t c_kuhn[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};
__constant__ int8_t c_kuhn_odd[6] = {0, 1, 1, 0, 0, 1};
// tetrahedron edges (vertex pairs in tetrahedron order)
__constant__ int8_t c_tet_edge[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
// triangles (tetrahedron edge triples) per inside pattern (bit v = tetrahedron vertex v inside), wound so that on a
// positively oriented tetrahedron the normal points from the inside vertices to the outside ones; two inside vertices
// i < j (outside k < l) give the quad (i,k) (i,l) (j,l) (j,k) split along (i,k)-(j,l)
__constant__ int8_t c_tris[16][2][3] = {
    {{-1, -1, -1}, {-1, -1, -1}}, {{0, 1, 2}, {-1, -1, -1}}, {{0, 4, 3}, {-1, -1, -1}}, {{1, 2, 4}, {1, 4, 3}},
    {{1, 3, 5}, {-1, -1, -1}},    {{0, 5, 2}, {0, 3, 5}},    {{0, 4, 5}, {0, 5, 1}},    {{2, 4, 5}, {-1, -1, -1}},
    {{2, 5, 4}, {-1, -1, -1}},    {{0, 1, 5}, {0, 5, 4}},    {{0, 5, 3}, {0, 2, 5}},    {{1, 5, 3}, {-1, -1, -1}},
    {{1, 3, 4}, {1, 4, 2}},       {{0, 3, 4}, {-1, -1, -1}}, {{0, 2, 1}, {-1, -1, -1}}, {{-1, -1, -1}, {-1, -1, -1}}};

struct IsoGrid {
  const float* v;
  int nx, ny, nz;
  float iso;
  int64_t n;  // nx ny nz
};

__device__ __forceinline__ int tris_of_pattern(int pat) {
  const int c = __popc(pat);
  return c == 2 ? 2 : (c & 1);
}

// The corners of point p's cell that exist (bit c of `valid`, c = x | y << 1 | z << 2) and which of them are inside.
__device__ __forceinline__ void cell_corners(const IsoGrid& g, int64_t p, int& i, int& j, int& k, uint32_t& valid,
                                             uint32_t& in, float (&val)[8]) {
  i = (int)(p % g.nx);
  const int64_t q = p / g.nx;
  j = (int)(q % g.ny);
  k = (int)(q / g.ny);
  valid = 0, in = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
    val[c] = 0.f;
    if (i + dx < g.nx && j + dy < g.ny && k + dz < g.nz) {
      val[c] = __ldg(g.v + p + dx + (int64_t)g.nx * (dy + (int64_t)g.ny * dz));
      valid |= 1u << c;
      if (val[c] > g.iso) in |= 1u << c;
    }
  }
}

// bit d: the edge of point p in direction d carries a vertex
__device__ __forceinline__ uint32_t edge_mask(uint32_t valid, uint32_t in) {
  uint32_t m = 0;
#pragma unroll
  for (int d = 0; d < 7; ++d) {
    const int b = c_bits_of_dir[d];
    if (((valid >> b) & 1u) && ((in ^ (in >> b)) & 1u)) m |= 1u << d;
  }
  return m;
}

// triangles of p's cell (0 when p is on the last layer of any axis)
__device__ __forceinline__ int cell_tris(const IsoGrid& g, int i, int j, int k, uint32_t in) {
  if (i + 1 >= g.nx || j + 1 >= g.ny || k + 1 >= g.nz) return 0;
  int f = 0;
#pragma unroll
  for (int t = 0; t < 6; ++t) {
    int pat = 0;
#pragma unroll
    for (int v = 0; v < 4; ++v) pat |= (int)((in >> c_kuhn[t][v]) & 1u) << v;
    f += tris_of_pattern(pat);
  }
  return f;
}

// exclusive scan over the block (kThreads threads) of one value per thread; `total` = the block's sum
template <int kThreads, typename T>
__device__ __forceinline__ T block_excl_scan(T v, T* warp_sums, T& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    T s = lane < kThreads / 32 ? warp_sums[lane] : T(0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T n = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += n;
    }
    if (lane < kThreads / 32) warp_sums[lane] = s;  // inclusive
  }
  __syncthreads();
  total = warp_sums[kThreads / 32 - 1];
  const T before = warp > 0 ? warp_sums[warp - 1] : T(0);
  __syncthreads();  // warp_sums is reused by the caller's next scan
  return before + inc - v;
}

// pass 1: vertices and triangles per tile
__global__ void __launch_bounds__(kIsoThreads) iso_count_kernel(const IsoGrid g, int64_t* __restrict__ tile_v,
                                                                int64_t* __restrict__ tile_f) {
  __shared__ int sums[kIsoThreads / 32];
  const int64_t p0 = (int64_t)blockIdx.x * kIsoTile + (int64_t)threadIdx.x * kIsoPer;
  int nv = 0, nf = 0;
  for (int e = 0; e < kIsoPer; ++e) {
    const int64_t p = p0 + e;
    if (p >= g.n) break;
    int i, j, k;
    uint32_t valid, in;
    float val[8];
    cell_corners(g, p, i, j, k, valid, in, val);
    nv += __popc(edge_mask(valid, in));
    nf += cell_tris(g, i, j, k, in);
  }
  int tv, tf;
  block_excl_scan<kIsoThreads>(nv, sums, tv);
  block_excl_scan<kIsoThreads>(nf, sums, tf);
  if (threadIdx.x == 0) tile_v[blockIdx.x] = tv, tile_f[blockIdx.x] = tf;
}

// tile counts -> exclusive tile offsets (in place), one block; totals[0..1] (and counts[0..1]) = vertices, faces
__global__ void __launch_bounds__(kScanThreads) iso_scan_kernel(int64_t* __restrict__ tile_v, int64_t* __restrict__ tile_f,
                                                                int64_t tiles, int64_t* __restrict__ totals,
                                                                int64_t* __restrict__ counts) {
  __shared__ long long sums[kScanThreads / 32];
  const int64_t per = (tiles + kScanThreads - 1) / kScanThreads;
  const int64_t b = (int64_t)threadIdx.x * per, e = b + per < tiles ? b + per : tiles;
  for (int a = 0; a < 2; ++a) {
    int64_t* arr = a == 0 ? tile_v : tile_f;
    long long s = 0;
    for (int64_t t = b; t < e; ++t) s += arr[t];
    long long total;
    long long run = block_excl_scan<kScanThreads>(s, sums, total);
    for (int64_t t = b; t < e; ++t) {
      const long long c = arr[t];
      arr[t] = run;
      run += c;
    }
    if (threadIdx.x == 0) {
      totals[a] = total;
      counts[a] = total;
    }
  }
}

__device__ __forceinline__ float lattice(float lo, float step, int idx) { return __fadd_rn(lo, __fmul_rn((float)idx, step)); }

struct IsoFrame {
  float lo[3], step[3];
};

// pass 2a: each point's edge mask and first vertex id, and its vertices
__global__ void __launch_bounds__(kIsoThreads) iso_vertex_kernel(const IsoGrid g, const IsoFrame fr,
                                                                 const int64_t* __restrict__ tile_v,
                                                                 uint8_t* __restrict__ mask, int32_t* __restrict__ vbase,
                                                                 float* __restrict__ verts) {
  __shared__ int sums[kIsoThreads / 32];
  const int64_t p0 = (int64_t)blockIdx.x * kIsoTile + (int64_t)threadIdx.x * kIsoPer;
  uint32_t m[kIsoPer];
  int nv = 0;
#pragma unroll
  for (int e = 0; e < kIsoPer; ++e) {
    m[e] = 0;
    const int64_t p = p0 + e;
    if (p < g.n) {
      int i, j, k;
      uint32_t valid, in;
      float val[8];
      cell_corners(g, p, i, j, k, valid, in, val);
      m[e] = edge_mask(valid, in);
      nv += __popc(m[e]);
    }
  }
  int total;
  int64_t id = tile_v[blockIdx.x] + block_excl_scan<kIsoThreads>(nv, sums, total);
  for (int e = 0; e < kIsoPer; ++e) {
    const int64_t p = p0 + e;
    if (p >= g.n) break;
    mask[p] = (uint8_t)m[e];
    vbase[p] = (int32_t)id;
    if (!m[e]) continue;
    int i, j, k;
    uint32_t valid, in;
    float val[8];
    cell_corners(g, p, i, j, k, valid, in, val);
    const int idx[3] = {i, j, k};
    for (int d = 0; d < 7; ++d) {
      if (!((m[e] >> d) & 1u)) continue;
      const int b = c_bits_of_dir[d];
      float t = __fdiv_rn(__fsub_rn(g.iso, val[0]), __fsub_rn(val[b], val[0]));
      if (t != t) t = 0.5f;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float pa = lattice(fr.lo[a], fr.step[a], idx[a]);
        const float pb = lattice(fr.lo[a], fr.step[a], idx[a] + ((b >> a) & 1));
        verts[id * 3 + a] = __fadd_rn(pa, __fmul_rn(t, __fsub_rn(pb, pa)));
      }
      ++id;
    }
  }
}

// pass 2b: the triangles of each cell
__global__ void __launch_bounds__(kIsoThreads) iso_face_kernel(const IsoGrid g, const int64_t* __restrict__ tile_f,
                                                               const uint8_t* __restrict__ mask,
                                                               const int32_t* __restrict__ vbase,
                                                               int32_t* __restrict__ faces) {
  __shared__ int sums[kIsoThreads / 32];
  const int64_t p0 = (int64_t)blockIdx.x * kIsoTile + (int64_t)threadIdx.x * kIsoPer;
  int nf = 0;
  for (int e = 0; e < kIsoPer; ++e) {
    const int64_t p = p0 + e;
    if (p >= g.n) break;
    int i, j, k;
    uint32_t valid, in;
    float val[8];
    cell_corners(g, p, i, j, k, valid, in, val);
    nf += cell_tris(g, i, j, k, in);
  }
  int total;
  int64_t f = tile_f[blockIdx.x] + block_excl_scan<kIsoThreads>(nf, sums, total);
  for (int e = 0; e < kIsoPer; ++e) {
    const int64_t p = p0 + e;
    if (p >= g.n) break;
    int i, j, k;
    uint32_t valid, in;
    float val[8];
    cell_corners(g, p, i, j, k, valid, in, val);
    if (cell_tris(g, i, j, k, in) == 0) continue;
    for (int t = 0; t < 6; ++t) {
      int pat = 0;
      for (int v = 0; v < 4; ++v) pat |= (int)((in >> c_kuhn[t][v]) & 1u) << v;
      for (int r = 0; r < 2; ++r) {
        if (c_tris[pat][r][0] < 0) break;
        int32_t ids[3];
        for (int q = 0; q < 3; ++q) {
          const int te = c_tris[pat][r][q];
          const int ca = c_kuhn[t][c_tet_edge[te][0]], cb = c_kuhn[t][c_tet_edge[te][1]];
          const int64_t owner = p + (ca & 1) + (int64_t)g.nx * (((ca >> 1) & 1) + (int64_t)g.ny * (ca >> 2));
          const int d = c_dir_of_bits[ca ^ cb];
          ids[q] = vbase[owner] + __popc((uint32_t)mask[owner] & ((1u << d) - 1u));
        }
        const bool flip = c_kuhn_odd[t];
        faces[f * 3 + 0] = ids[0];
        faces[f * 3 + 1] = ids[flip ? 2 : 1];
        faces[f * 3 + 2] = ids[flip ? 1 : 2];
        ++f;
      }
    }
  }
}

// d(grid)/d(axis a) at lattice point idx (p its flat index): (v[+1] - v[-1]) / (2 step) inside, one-sided over step at
// the box faces
__device__ __forceinline__ float grid_partial(const IsoGrid& g, int64_t p, const int (&idx)[3], int a, float step) {
  const int n = a == 0 ? g.nx : (a == 1 ? g.ny : g.nz);
  const int64_t stride = a == 0 ? 1 : (a == 1 ? (int64_t)g.nx : (int64_t)g.nx * g.ny);
  const bool lo = idx[a] == 0, hi = idx[a] == n - 1;
  const float vp = __ldg(g.v + (hi ? p : p + stride)), vm = __ldg(g.v + (lo ? p : p - stride));
  return __fdiv_rn(__fsub_rn(vp, vm), (lo || hi) ? step : __fmul_rn(2.f, step));
}

// pass 3 (after pass 2a): vertex normals, in the vertex order of iso_vertex_kernel (one thread per lattice point)
__global__ void __launch_bounds__(kIsoThreads) iso_normal_kernel(const IsoGrid g, const IsoFrame fr,
                                                                 const uint8_t* __restrict__ mask,
                                                                 const int32_t* __restrict__ vbase,
                                                                 float* __restrict__ normals) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= g.n) return;
  const uint32_t m = mask[p];
  if (!m) return;
  int64_t id = vbase[p];
  const int i = (int)(p % g.nx);
  const int64_t q = p / g.nx;
  const int j = (int)(q % g.ny), k = (int)(q / g.ny);
  const int ia[3] = {i, j, k};
  const float va = __ldg(g.v + p);
  float ga[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) ga[a] = grid_partial(g, p, ia, a, fr.step[a]);
  for (int d = 0; d < 7; ++d) {
    if (!((m >> d) & 1u)) continue;
    const int b = c_bits_of_dir[d];
    const int ib[3] = {i + (b & 1), j + ((b >> 1) & 1), k + (b >> 2)};
    const int64_t pb = p + (b & 1) + (int64_t)g.nx * (((b >> 1) & 1) + (int64_t)g.ny * (b >> 2));
    const float vb = __ldg(g.v + pb);
    float t = __fdiv_rn(__fsub_rn(g.iso, va), __fsub_rn(vb, va));  // the vertex's t (iso_vertex_kernel)
    if (t != t) t = 0.5f;
    float n[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float gb = grid_partial(g, pb, ib, a, fr.step[a]);
      n[a] = __fadd_rn(ga[a], __fmul_rn(t, __fsub_rn(gb, ga[a])));
    }
    const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2])));
    const bool ok = len > 0.f && len < INFINITY;  // false for NaN too
#pragma unroll
    for (int a = 0; a < 3; ++a) normals[id * 3 + a] = ok ? __fdiv_rn(-n[a], len) : 0.f;
    ++id;
  }
}

// scratch: [totals 2] [tile_v tiles] [tile_f tiles] (int64) | vbase [n] int32 | mask [n] uint8
struct IsoScratch {
  int64_t *totals, *tile_v, *tile_f;
  int32_t* vbase;
  uint8_t* mask;
  int64_t tiles;
  size_t bytes;
};
inline size_t iso_align(size_t v) { return (v + 255) / 256 * 256; }
IsoScratch carve_iso(int nx, int ny, int nz, void* base) {
  IsoScratch s{};
  const int64_t n = (int64_t)nx * ny * nz;
  s.tiles = (n + kIsoTile - 1) / kIsoTile;
  uint8_t* b = static_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = b ? b + off : nullptr;
    off += iso_align(bytes);
    return p;
  };
  s.totals = reinterpret_cast<int64_t*>(take((size_t)(2 + 2 * s.tiles) * sizeof(int64_t)));
  s.tile_v = s.totals ? s.totals + 2 : nullptr;
  s.tile_f = s.totals ? s.totals + 2 + s.tiles : nullptr;
  s.vbase = reinterpret_cast<int32_t*>(take((size_t)n * sizeof(int32_t)));
  s.mask = take((size_t)n);
  s.bytes = off;
  return s;
}

}  // namespace

size_t isosurface_scratch_bytes(int nx, int ny, int nz) { return carve_iso(nx, ny, nz, nullptr).bytes; }

const int64_t* isosurface_totals(const void* scratch) { return static_cast<const int64_t*>(scratch); }

cudaError_t launch_isosurface_count(const float* grid, int nx, int ny, int nz, float iso, void* scratch,
                                    int64_t* counts, cudaStream_t st) {
  const IsoScratch s = carve_iso(nx, ny, nz, scratch);
  const IsoGrid g{grid, nx, ny, nz, iso, (int64_t)nx * ny * nz};
  LaunchScope scope(kKernIsosurface, st);
  iso_count_kernel<<<(unsigned)s.tiles, kIsoThreads, 0, st>>>(g, s.tile_v, s.tile_f);
  iso_scan_kernel<<<1, kScanThreads, 0, st>>>(s.tile_v, s.tile_f, s.tiles, s.totals, counts);
  return cudaGetLastError();
}

cudaError_t launch_isosurface_emit(const float* grid, int nx, int ny, int nz, const float* lo, const float* step,
                                   float iso, const void* scratch, float* verts, int32_t* faces, cudaStream_t st) {
  const IsoScratch s = carve_iso(nx, ny, nz, const_cast<void*>(scratch));
  const IsoGrid g{grid, nx, ny, nz, iso, (int64_t)nx * ny * nz};
  IsoFrame fr;
  for (int a = 0; a < 3; ++a) fr.lo[a] = lo[a], fr.step[a] = step[a];
  LaunchScope scope(kKernIsosurface, st);
  iso_vertex_kernel<<<(unsigned)s.tiles, kIsoThreads, 0, st>>>(g, fr, s.tile_v, s.mask, s.vbase, verts);
  iso_face_kernel<<<(unsigned)s.tiles, kIsoThreads, 0, st>>>(g, s.tile_f, s.mask, s.vbase, faces);
  return cudaGetLastError();
}

cudaError_t launch_isosurface_normals(const float* grid, int nx, int ny, int nz, const float* step, float iso,
                                      const void* scratch, float* normals, cudaStream_t st) {
  const IsoScratch s = carve_iso(nx, ny, nz, const_cast<void*>(scratch));
  const IsoGrid g{grid, nx, ny, nz, iso, (int64_t)nx * ny * nz};
  IsoFrame fr;
  for (int a = 0; a < 3; ++a) fr.lo[a] = 0.f, fr.step[a] = step[a];
  LaunchScope scope(kKernIsosurface, st);
  iso_normal_kernel<<<(unsigned)((g.n + kIsoThreads - 1) / kIsoThreads), kIsoThreads, 0, st>>>(g, fr, s.mask, s.vbase,
                                                                                                normals);
  return cudaGetLastError();
}

}  // namespace mipnerf
