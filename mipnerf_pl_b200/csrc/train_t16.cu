// train_t16.cu — the backward pass of the tensor-core training step on 16-bit "tile images".
//
// The training forward (mlp_tc.cu, mlp_level_kernel with an activation dump) leaves every activation in HBM exactly as the tensor
// core consumed it: per 128-row tile (= one ray's samples) and 64-column slab a [128 x 128 B] block in the
// 128-byte-swizzle layout (tc::sw128_offset), the slabs of a tile contiguous.  Everything here reads and writes that
// format, so operand staging is one cp.async.bulk per slab — no conversion, no register staging:
//   linear_t16_kernel     dX = [mask > 0] * (dY . B^T + r1[row] * r1w[col])        the dgrad chain, wgmma
//   color_dgrad_t16       d v = [v > 0] * (d raw_rgb @ Wc)                           colour head -> view layer
//   wgrad_small_n_t16     partials of dY^T X for the two narrow heads (n = 1, 3)     X = tile image, dY fp32
//   t16_pack / t16_unpack fp32 row-major <-> tile image (tests, stand-alone entry points)
// The wgrad GEMMs on tile images are in linear_tc.cu (wgrad_mn_kernel: a row-major tile IS an MN-major operand).
#include "kernels.h"
#include "mlp_tc.h"
#include "profile.h"
#include "ray_math.cuh"
#include "tc_common.cuh"

namespace mipnerf {
namespace {

using namespace tc;

constexpr uint32_t kSlab = 16384;  // [128 rows x 64 cols] 16-bit

// one 32-byte sector per thread, as two 128-bit accesses
__device__ __forceinline__ void ldg256(const void* p, uint32_t (&v)[8]) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(p)), b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
  v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
}
__device__ __forceinline__ void stg256(void* p, const uint32_t (&v)[8]) {
  reinterpret_cast<uint4*>(p)[0] = make_uint4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(v[4], v[5], v[6], v[7]);
}

struct LinearT16Params {
  const uint8_t* x;      // [tiles][k / 64][16 KB]
  const uint8_t* image;  // packed B: [k / 64][n x 128 B]   (pack_linear_image_kernel)
  uint8_t* y;            // [tiles][n / 64][16 KB]
  const uint8_t* mask;   // like y, or null: output zeroed where mask <= 0 (ReLU backward)
  const uint8_t* mask_bits;  // or the same mask as sign bits, [tiles * 128][32 B] (n = 256)
  const float* r1;       // [tiles * 128] or null, with r1w [n]: + r1[row] * r1w[col]  (density head)
  const float* r1w;
  int64_t tiles;
  int n, k;
};

// 256 threads = two warpgroups, persistent over 128-row tiles.  Thread 0 fetches the whole B image once and each
// tile's A slabs by cp.async.bulk; warpgroup g runs the wgmma of rows 64 g .. 64 g + 63 over N in 128-column chunks and
// writes the epilogue from its register accumulators straight into the output tile image.
template <int kFmt>
__global__ void __launch_bounds__(256, 1) linear_t16_kernel(const LinearT16Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  const int slabs = p.k >> 6;
  uint8_t* sA = smem;
  uint8_t* sB = sA + (size_t)slabs * kSlab;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + (size_t)slabs * p.n * 128);
  uint64_t* bar_b = bars;
  uint64_t* a_full = bars + 1;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, wq = warp & 3;
  if (tid == 0) {
    mbar_init(bar_b, 1);
    mbar_init(a_full, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_b, (uint32_t)(slabs * p.n * 128));
    for (int s = 0; s < slabs; ++s)
      bulk_g2s(sB + (size_t)s * p.n * 128, p.image + (size_t)s * p.n * 128, (uint32_t)(p.n * 128), bar_b);
  }
  mbar_wait(bar_b, 0);
  const int y_slabs = p.n >> 6;
  const uint32_t a_u = smem_u32(sA) + (uint32_t)wg * 8192u, b_u = smem_u32(sB);
  int it = 0;
  for (int64_t tile = blockIdx.x; tile < p.tiles; tile += gridDim.x, ++it) {
    if (tid == 0) {
      mbar_arrive_expect_tx(a_full, (uint32_t)slabs * kSlab);
      for (int s = 0; s < slabs; ++s)
        bulk_g2s(sA + (size_t)s * kSlab, p.x + ((size_t)tile * slabs + s) * kSlab, kSlab, a_full);
    }
    mbar_wait(a_full, (uint32_t)it & 1u);
    uint8_t* ytile = p.y + (size_t)tile * y_slabs * kSlab;
    const uint8_t* mtile = p.mask ? p.mask + (size_t)tile * y_slabs * kSlab : nullptr;
    const int r_lo = 64 * wg + 16 * wq + (lane >> 2);
    for (int nc = 0; nc < p.n; nc += 128) {
      float acc[64];
      wgmma_fence_acc(acc);
      wgmma_fence();
      for (int s = 0; s < slabs; ++s)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          wgmma_m64n128k16<kFmt>(acc, make_sw128_desc(a_u + (uint32_t)s * kSlab + 32u * j),
                                 make_sw128_desc(b_u + (uint32_t)(s * p.n + nc) * 128u + 32u * j), (s | j) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r_lo + 8 * h;
        const float rv = p.r1 ? __ldg(p.r1 + tile * 128 + row) : 0.f;
        const uint8_t* mb = p.mask_bits ? p.mask_bits + ((size_t)tile * 128 + row) * 32 : nullptr;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = nc + 8 * j + 2 * (lane & 3);
          float o0 = acc[4 * j + 2 * h], o1 = acc[4 * j + 2 * h + 1];
          if (p.r1) {
            const float2 w = __ldg(reinterpret_cast<const float2*>(p.r1w + col));
            o0 = fmaf(rv, w.x, o0), o1 = fmaf(rv, w.y, o1);
          }
          const uint32_t off = (uint32_t)(col >> 6) * kSlab + sw128_offset(row, col & 63);
          if (mtile) {  // a 16-bit float is > 0 iff its bits, read as a signed integer, are > 0
            const uint32_t mw = __ldg(reinterpret_cast<const uint32_t*>(mtile + off));
            if (!((int16_t)(mw & 0xffffu) > 0)) o0 = 0.f;
            if (!((int32_t)mw >= 0x00010000)) o1 = 0.f;
          } else if (mb) {  // bit (column % 8) of byte (column / 8)
            const uint32_t byte = __ldg(mb + (col >> 3));
            if (!((byte >> (col & 7)) & 1u)) o0 = 0.f;
            if (!((byte >> ((col & 7) + 1)) & 1u)) o1 = 0.f;
          }
          *reinterpret_cast<uint32_t*>(ytile + off) = pack2<kFmt>(o0, o1);
        }
      }
    }
    __syncthreads();  // both warpgroups' wgmmas are done with the A slabs before the next tile's copy
  }
}

// The split-operand (bf16x3) dgrad: x = x_hi + x_lo and B = B_hi + B_lo, each K-step x_hi.B_hi + x_lo.B_hi + x_hi.B_lo
// into one fp32 accumulator (the level kernel's order; x_lo.B_lo, below 2^-16 relative, is dropped), the output written
// as y_hi = fl16(y) and y_lo = fl16(y - y_hi).  Hi + lo copies of the layout above would take 384 KB, so a CTA owns one
// 128-column N-half for good and keeps that half of B, hi and lo, resident: 2 x k/64 x 16 KB = 128 KB at k = 256.  A
// streams per 64-wide K-slab, hi + lo = 32 KB, through a two-slot ring: 64 KB.  192 KB in all at n = k = 256 (plus the
// 1 KB alignment slack and the mbarriers).  Warps 0-7 are the two wgmma warpgroups (rows 64 g ..), warp 8 issues the
// bulk copies.
struct LinearT16X3Params {
  LinearT16Params hi;  // x, image, y: the hi images; mask / mask_bits / r1 as for linear_t16_kernel
  const uint8_t* x_lo;
  const uint8_t* image_lo;
  uint8_t* y_lo;
};

template <int kFmt>
__global__ void __launch_bounds__(288, 1) linear_t16_x3_kernel(const LinearT16X3Params q) {
  const LinearT16Params& p = q.hi;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  const int slabs = p.k >> 6, halves = p.n >> 7;
  uint8_t* sB = smem;                                       // [hi, lo][slabs][128 rows x 128 B]
  uint8_t* sA = sB + (size_t)2 * slabs * kSlab;             // [2 slots][hi, lo][16 KB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sA + 4 * kSlab);
  uint64_t* bar_b = bars;
  uint64_t* full = bars + 1;   // [2] producer (tx bytes) -> warpgroups
  uint64_t* empty = bars + 3;  // [2] one arrive per warpgroup once its wgmmas have read the slot
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nc = 128 * (int)(blockIdx.x % halves);
  const int64_t tile0 = blockIdx.x / halves, tstep = gridDim.x / halves;
  if (tid == 0) {
    mbar_init(bar_b, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (warp == 8) {
    if (lane == 0) {
      mbar_arrive_expect_tx(bar_b, (uint32_t)(2 * slabs) * kSlab);
      for (int s = 0; s < slabs; ++s) {
        const size_t src = ((size_t)s * p.n + nc) * 128;
        bulk_g2s(sB + (size_t)s * kSlab, p.image + src, kSlab, bar_b);
        bulk_g2s(sB + (size_t)(slabs + s) * kSlab, q.image_lo + src, kSlab, bar_b);
      }
      int it = 0;
      for (int64_t tile = tile0; tile < p.tiles; tile += tstep)
        for (int s = 0; s < slabs; ++s, ++it) {
          const int b = it & 1;
          if (it >= 2) mbar_wait(&empty[b], (uint32_t)((it >> 1) - 1) & 1u);
          mbar_arrive_expect_tx(&full[b], 2 * kSlab);
          const size_t src = ((size_t)tile * slabs + s) * kSlab;
          bulk_g2s(sA + (size_t)(2 * b) * kSlab, p.x + src, kSlab, &full[b]);
          bulk_g2s(sA + (size_t)(2 * b + 1) * kSlab, q.x_lo + src, kSlab, &full[b]);
        }
    }
    return;
  }
  const int wg = warp >> 2, wq = warp & 3;
  const bool leader = (tid & 127) == 0;
  const int r_lo = 64 * wg + 16 * wq + (lane >> 2);
  const int y_slabs = p.n >> 6;
  const uint32_t a_u = smem_u32(sA) + (uint32_t)wg * 8192u, b_u = smem_u32(sB);
  const uint32_t b_lo = (uint32_t)slabs * kSlab / 16u;  // descriptor offsets of the lo operands
  constexpr uint32_t a_lo = kSlab / 16u;
  mbar_wait(bar_b, 0);
  int it = 0;
  for (int64_t tile = tile0; tile < p.tiles; tile += tstep) {
    float acc[64];
    wgmma_fence_acc(acc);
    for (int s = 0; s < slabs; ++s, ++it) {
      const int b = it & 1;
      mbar_wait(&full[b], (uint32_t)(it >> 1) & 1u);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint64_t ad = make_sw128_desc(a_u + (uint32_t)(2 * b) * kSlab + 32u * j);
        const uint64_t bd = make_sw128_desc(b_u + (uint32_t)s * kSlab + 32u * j);
        wgmma_m64n128k16<kFmt>(acc, ad, bd, (s | j) ? 1u : 0u);
        wgmma_m64n128k16<kFmt>(acc, ad + a_lo, bd, 1u);
        wgmma_m64n128k16<kFmt>(acc, ad, bd + b_lo, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (leader) mbar_arrive(&empty[b]);
    }
    uint8_t* ytile = p.y + (size_t)tile * y_slabs * kSlab;
    uint8_t* ltile = q.y_lo + (size_t)tile * y_slabs * kSlab;
    const uint8_t* mtile = p.mask ? p.mask + (size_t)tile * y_slabs * kSlab : nullptr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r_lo + 8 * h;
      const float rv = p.r1 ? __ldg(p.r1 + tile * 128 + row) : 0.f;
      const uint8_t* mb = p.mask_bits ? p.mask_bits + ((size_t)tile * 128 + row) * 32 : nullptr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = nc + 8 * j + 2 * (lane & 3);
        float o0 = acc[4 * j + 2 * h], o1 = acc[4 * j + 2 * h + 1];
        if (p.r1) {
          const float2 w = __ldg(reinterpret_cast<const float2*>(p.r1w + col));
          o0 = fmaf(rv, w.x, o0), o1 = fmaf(rv, w.y, o1);
        }
        const uint32_t off = (uint32_t)(col >> 6) * kSlab + sw128_offset(row, col & 63);
        if (mtile) {  // the hi image's sign: fl16(x) > 0 iff x > 0
          const uint32_t mw = __ldg(reinterpret_cast<const uint32_t*>(mtile + off));
          if (!((int16_t)(mw & 0xffffu) > 0)) o0 = 0.f;
          if (!((int32_t)mw >= 0x00010000)) o1 = 0.f;
        } else if (mb) {
          const uint32_t byte = __ldg(mb + (col >> 3));
          if (!((byte >> (col & 7)) & 1u)) o0 = 0.f;
          if (!((byte >> ((col & 7) + 1)) & 1u)) o1 = 0.f;
        }
        const uint32_t hv = pack2<kFmt>(o0, o1);
        *reinterpret_cast<uint32_t*>(ytile + off) = hv;
        *reinterpret_cast<uint32_t*>(ltile + off) = pack2_low<kFmt>(o0, o1, hv);
      }
    }
  }
}

// d v[row][c] = [v[row][c] > 0] * sum_j d_rgb[row][j] * wc[j][c]      thread = (row, 8-column chunk), k_dim = 128
// kX3: v is the hi image (its sign is v's), d v goes out as hi and lo images
template <int kFmt, bool kX3 = false>
__global__ void color_dgrad_t16_kernel(const float* __restrict__ d_rgb, const float* __restrict__ wc,
                                       const uint8_t* __restrict__ v, uint8_t* __restrict__ d_v, int64_t m,
                                       int k_dim, uint8_t* __restrict__ d_v_lo = nullptr) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int chunks = k_dim >> 3;
  if (idx >= m * chunks) return;
  const int64_t row = idx / chunks;
  const int ch = (int)(idx % chunks);
  const int r = (int)(row & 127);
  const size_t off = ((size_t)(row >> 7) * (k_dim >> 6) + (ch >> 3)) * kSlab + (uint32_t)r * 128u +
                     ((((uint32_t)ch & 7u) ^ ((uint32_t)r & 7u)) << 4);
  const float g0 = __ldg(d_rgb + row * 3), g1 = __ldg(d_rgb + row * 3 + 1), g2 = __ldg(d_rgb + row * 3 + 2);
  const uint4 mk = __ldg(reinterpret_cast<const uint4*>(v + off));
  const uint32_t mw[4] = {mk.x, mk.y, mk.z, mk.w};
  float o[8];
#pragma unroll
  for (int h = 0; h < 2; ++h) {  // Wc rows as float4 (six 16-byte loads instead of 24 scalar ones)
    const int c = ch * 8 + 4 * h;
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(wc + c));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(wc + k_dim + c));
    const float4 w2 = __ldg(reinterpret_cast<const float4*>(wc + 2 * k_dim + c));
    o[4 * h + 0] = fmaf(g2, w2.x, fmaf(g1, w1.x, g0 * w0.x));
    o[4 * h + 1] = fmaf(g2, w2.y, fmaf(g1, w1.y, g0 * w0.y));
    o[4 * h + 2] = fmaf(g2, w2.z, fmaf(g1, w1.z, g0 * w0.z));
    o[4 * h + 3] = fmaf(g2, w2.w, fmaf(g1, w1.w, g0 * w0.w));
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (!((int16_t)(mw[e] & 0xffffu) > 0)) o[2 * e] = 0.f;
    if (!((int32_t)mw[e] >= 0x00010000)) o[2 * e + 1] = 0.f;
  }
  if constexpr (kX3) {
    uint32_t hv[4], lv[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      hv[e] = pack2<kFmt>(o[2 * e], o[2 * e + 1]);
      lv[e] = pack2_low<kFmt>(o[2 * e], o[2 * e + 1], hv[e]);
    }
    *reinterpret_cast<uint4*>(d_v + off) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
    *reinterpret_cast<uint4*>(d_v_lo + off) = make_uint4(lv[0], lv[1], lv[2], lv[3]);
  } else {
    *reinterpret_cast<uint4*>(d_v + off) =
        make_uint4(pack2<kFmt>(o[0], o[1]), pack2<kFmt>(o[2], o[3]), pack2<kFmt>(o[4], o[5]), pack2<kFmt>(o[6], o[7]));
  }
}

template <int kFmt>
__device__ __forceinline__ float t16_load(const uint8_t* base, int64_t row, int col, int cols) {
  const uint16_t bits = __ldg(reinterpret_cast<const uint16_t*>(
      base + ((size_t)(row >> 7) * (cols >> 6) + (col >> 6)) * kSlab + sw128_offset((int)(row & 127), col & 63)));
  return from16<kFmt>(bits);
}

// The two narrow heads' weight gradients (density n = 1, colour n = 3) with X read from a tile image: an HBM-bound
// streaming pass.  A warp (k_dim = 256) or half-warp (128) owns a row at a time, each lane one 16-byte chunk (8 columns,
// coalesced 512 / 256 B per row), eight rows in flight per lane; the dY values of the row are warp-uniform fp32 loads.
// Lane partials are combined through shared memory in a fixed order; same partial layout as wgrad_small_n_kernel.
// kX3: X = hi + lo (x_lo the lo image), the two halves summed in fp32.
template <int kFmt, int kN, bool kX3 = false>
__global__ void __launch_bounds__(256)
wgrad_small_n_t16_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ x, int k_dim,
                         float* __restrict__ part, int64_t m, int64_t slice_rows,
                         const uint8_t* __restrict__ x_lo = nullptr) {
  __shared__ float red[8][32][kN * 8 + 1];
  __shared__ float bred[16][kN];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cpr = k_dim >> 3;        // 16-byte chunks per row: 32 or 16
  const int rpw = 32 / cpr;          // rows a warp covers per step: 1 or 2
  const int sub = lane / cpr, chunk = lane % cpr;
  const int64_t m_begin = (int64_t)blockIdx.x * slice_rows;
  const int64_t m_end = (m_begin + slice_rows) < m ? (m_begin + slice_rows) : m;
  float acc[kN][8], bsum[kN];
#pragma unroll
  for (int j = 0; j < kN; ++j) {
    bsum[j] = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[j][e] = 0.f;
  }
  const size_t slab_off = (size_t)(chunk >> 3) * kSlab;
  const uint32_t ci = (uint32_t)chunk & 7u;
  const int step = 8 * rpw;
  for (int64_t row0 = m_begin + warp * rpw + sub; row0 < m_end; row0 += (int64_t)step * 8) {
    uint4 xv[8], xl[8];
    float d[8][kN];
#pragma unroll
    for (int u = 0; u < 8; ++u) {  // eight independent rows in flight
      const int64_t row = row0 + (int64_t)u * step;
      const bool ok = row < m_end;
      const int r = (int)(row & 127);
      const size_t xo = (size_t)(row >> 7) * (cpr >> 3) * kSlab + slab_off + (uint32_t)r * 128u +
                        ((ci ^ ((uint32_t)r & 7u)) << 4);
      xv[u] = ok ? __ldg(reinterpret_cast<const uint4*>(x + xo)) : make_uint4(0u, 0u, 0u, 0u);
      if (kX3) xl[u] = ok ? __ldg(reinterpret_cast<const uint4*>(x_lo + xo)) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
      for (int j = 0; j < kN; ++j) d[u][j] = ok ? __ldg(dy + row * kN + j) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const uint32_t w[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
      const uint32_t wl[4] = {kX3 ? xl[u].x : 0u, kX3 ? xl[u].y : 0u, kX3 ? xl[u].z : 0u, kX3 ? xl[u].w : 0u};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float x0 = from16<kFmt>((uint16_t)(w[e] & 0xffffu)), x1 = from16<kFmt>((uint16_t)(w[e] >> 16));
        if (kX3) {
          x0 += from16<kFmt>((uint16_t)(wl[e] & 0xffffu));
          x1 += from16<kFmt>((uint16_t)(wl[e] >> 16));
        }
#pragma unroll
        for (int j = 0; j < kN; ++j) {
          acc[j][2 * e] = fmaf(d[u][j], x0, acc[j][2 * e]);
          acc[j][2 * e + 1] = fmaf(d[u][j], x1, acc[j][2 * e + 1]);
        }
      }
#pragma unroll
      for (int j = 0; j < kN; ++j) bsum[j] += d[u][j];
    }
  }
#pragma unroll
  for (int j = 0; j < kN; ++j)
#pragma unroll
    for (int e = 0; e < 8; ++e) red[warp][lane][j * 8 + e] = acc[j][e];
  if (chunk == 0)
#pragma unroll
    for (int j = 0; j < kN; ++j) bred[warp * 2 + sub][j] = bsum[j];
  __syncthreads();
  float* out = part + (size_t)blockIdx.x * kN * (k_dim + 1);
  if (tid < k_dim) {  // column tid = chunk tid / 8, element tid % 8: fixed-order sum over warps and sub-rows
    const int c = tid >> 3, e = tid & 7;
#pragma unroll
    for (int j = 0; j < kN; ++j) {
      float v = 0.f;
      for (int w8 = 0; w8 < 8; ++w8)
        for (int sb = 0; sb < rpw; ++sb) v += red[w8][sb * cpr + c][j * 8 + e];
      out[(size_t)j * (k_dim + 1) + tid] = v;
    }
  }
  if (tid < kN) {
    float v = 0.f;
    for (int w8 = 0; w8 < 8; ++w8)
      for (int sb = 0; sb < rpw; ++sb) v += bred[w8 * 2 + sb][tid];
    out[(size_t)tid * (k_dim + 1) + k_dim] = v;
  }
}

// The 96 IPE features of every sample as a tile image [rays][2 slabs] (columns 96..127 zero): the X operand of the
// layer-0 / skip-layer wgrads.  Same device functions and the same MUFU fast path as the level kernel's IPE warps
// (mlp_tc.cu: ipe_row_group), so these are bit for bit the features the forward multiplied with.  Thread = (sample row,
// k): k < 6 computes the Gaussian once and the eight (degree, coordinate) pairs 8k..8k+7, i.e. sin chunk k and cos
// chunk 6 + k; k = 6, 7 zero the padding chunks.
// kX3: hi and lo images (out_lo), split as the split level kernel's feature tile (mlp_tc.cu: store8_split).
template <int kFmt, bool kX3 = false>
__global__ void __launch_bounds__(256) ipe_t16_kernel(const float* __restrict__ origins,
                                                      const float* __restrict__ directions,
                                                      const float* __restrict__ radii, const float* __restrict__ t,
                                                      uint8_t* __restrict__ out, int64_t num_rays, int n,
                                                      int disable_integration, uint8_t* __restrict__ out_lo = nullptr) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= num_rays * n * 8) return;
  const int64_t p = idx >> 3;  // sample index = ray * n + j   (n = 128: tile = ray, row = j)
  const int k = (int)(idx & 7);
  const int r = (int)(p & 127);
  const size_t tile_off = (size_t)(p >> 7) * (2 * kSlab) + (uint32_t)r * 128u;
  uint8_t* tile = out + tile_off;
  const uint32_t rx = (uint32_t)r & 7u;
  auto chunk_off = [&](int ch) { return (size_t)(ch >> 3) * kSlab + ((((uint32_t)ch & 7u) ^ rx) << 4); };
  auto chunk_ptr = [&](int ch) { return tile + chunk_off(ch); };
  if (k >= 6) {
    *reinterpret_cast<uint4*>(chunk_ptr(12 + 2 * (k - 6))) = make_uint4(0u, 0u, 0u, 0u);
    *reinterpret_cast<uint4*>(chunk_ptr(13 + 2 * (k - 6))) = make_uint4(0u, 0u, 0u, 0u);
    if (kX3) {
      *reinterpret_cast<uint4*>(out_lo + tile_off + chunk_off(12 + 2 * (k - 6))) = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(out_lo + tile_off + chunk_off(13 + 2 * (k - 6))) = make_uint4(0u, 0u, 0u, 0u);
    }
    return;
  }
  const int64_t ray = p / n;
  const int j = (int)(p % n);
  const RayGeom g = load_ray_geom(origins, directions, radii, ray);
  const float t0 = __ldg(t + ray * (n + 1) + j), t1 = __ldg(t + ray * (n + 1) + j + 1);
  float tm, tv, rv, mean[3], cov[3];
  frustum_moments(t0, t1, g.radius_sq, tm, tv, rv);
  lift_gaussian(g, tm, tv, rv, mean, cov);
  if (disable_integration) cov[0] = cov[1] = cov[2] = 0.f;
  float fs[8], fc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int f = k * 8 + e;  // feature index = degree * 3 + coord   (models/mip.py:335-341)
    ipe_pair<true>(mean[f % 3], cov[f % 3], f / 3, fs[e], fc[e]);
  }
  if constexpr (kX3) {
    auto split8 = [&](const float (&v)[8], size_t o) {
      uint32_t hv[4], lv[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        hv[e] = pack2<kFmt>(v[2 * e], v[2 * e + 1]);
        lv[e] = pack2_low<kFmt>(v[2 * e], v[2 * e + 1], hv[e]);
      }
      *reinterpret_cast<uint4*>(out + tile_off + o) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
      *reinterpret_cast<uint4*>(out_lo + tile_off + o) = make_uint4(lv[0], lv[1], lv[2], lv[3]);
    };
    split8(fs, chunk_off(k));
    split8(fc, chunk_off(6 + k));
    return;
  }
  *reinterpret_cast<uint4*>(chunk_ptr(k)) =
      make_uint4(pack2<kFmt>(fs[0], fs[1]), pack2<kFmt>(fs[2], fs[3]), pack2<kFmt>(fs[4], fs[5]), pack2<kFmt>(fs[6], fs[7]));
  *reinterpret_cast<uint4*>(chunk_ptr(6 + k)) =
      make_uint4(pack2<kFmt>(fc[0], fc[1]), pack2<kFmt>(fc[2], fc[3]), pack2<kFmt>(fc[4], fc[5]), pack2<kFmt>(fc[6], fc[7]));
}

// The sibling for query points (the backward of the level kernel's query modes): row p of the image is the IPE of
// Gaussian p of means / covs [num_points, 3] (covs null or disable_integration: zero covariance), with ipe_pair<false>
// as the query modes' helper warps (mlp_tc.cu: ipe_row_group<.., kDensity = true>) compute it, so these are bit for bit
// the features the query multiplied with.  Rows past num_points up to the last whole tile are the IPE of a zero
// Gaussian, as in the query's feature tile: finite.  Thread layout as ipe_t16_kernel.
template <int kFmt>
__global__ void __launch_bounds__(256) ipe_points_t16_kernel(const float* __restrict__ means,
                                                             const float* __restrict__ covs, uint8_t* __restrict__ out,
                                                             int64_t num_points, int64_t padded_rows,
                                                             int disable_integration) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= padded_rows * 8) return;
  const int64_t p = idx >> 3;
  const int k = (int)(idx & 7);
  const int r = (int)(p & 127);
  uint8_t* tile = out + (size_t)(p >> 7) * (2 * kSlab) + (uint32_t)r * 128u;
  const uint32_t rx = (uint32_t)r & 7u;
  auto chunk_ptr = [&](int ch) { return tile + (size_t)(ch >> 3) * kSlab + ((((uint32_t)ch & 7u) ^ rx) << 4); };
  if (k >= 6) {
    *reinterpret_cast<uint4*>(chunk_ptr(12 + 2 * (k - 6))) = make_uint4(0u, 0u, 0u, 0u);
    *reinterpret_cast<uint4*>(chunk_ptr(13 + 2 * (k - 6))) = make_uint4(0u, 0u, 0u, 0u);
    return;
  }
  float mean[3] = {0.f, 0.f, 0.f}, cov[3] = {0.f, 0.f, 0.f};
  if (p < num_points) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      mean[c] = __ldg(means + p * 3 + c);
      cov[c] = covs && !disable_integration ? __ldg(covs + p * 3 + c) : 0.f;
    }
  }
  float fs[8], fc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int f = k * 8 + e;  // feature index = degree * 3 + coord   (models/mip.py:335-341)
    ipe_pair<false>(mean[f % 3], cov[f % 3], f / 3, fs[e], fc[e]);
  }
  *reinterpret_cast<uint4*>(chunk_ptr(k)) =
      make_uint4(pack2<kFmt>(fs[0], fs[1]), pack2<kFmt>(fs[2], fs[3]), pack2<kFmt>(fs[4], fs[5]), pack2<kFmt>(fs[6], fs[7]));
  *reinterpret_cast<uint4*>(chunk_ptr(6 + k)) =
      make_uint4(pack2<kFmt>(fc[0], fc[1]), pack2<kFmt>(fc[2], fc[3]), pack2<kFmt>(fc[4], fc[5]), pack2<kFmt>(fc[6], fc[7]));
}

// fp32 row-major [m, cols] (ld) <-> tile image; rows beyond m / columns beyond cols are zero in the image.
// thread = (row, 16-byte chunk of 8 columns): two float4 loads when the source allows it, one 16-byte store
template <int kFmt>
__global__ void t16_pack_kernel(const float* __restrict__ src, int ld, int cols, int64_t m, uint8_t* __restrict__ dst,
                                int img_cols, int64_t padded_rows, int vec, uint8_t* __restrict__ dst_lo) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int chunks = img_cols >> 3;
  if (idx >= padded_rows * chunks) return;
  const int64_t row = idx / chunks;
  const int ch = (int)(idx % chunks), c0 = ch * 8;
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (row < m) {
    if (vec && c0 + 8 <= cols) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(src + row * ld + c0));
      const float4 b = __ldg(reinterpret_cast<const float4*>(src + row * ld + c0 + 4));
      v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (c0 + e < cols) v[e] = __ldg(src + row * ld + c0 + e);
    }
  }
  const int r = (int)(row & 127);
  const size_t o = ((size_t)(row >> 7) * (img_cols >> 6) + (ch >> 3)) * kSlab + (uint32_t)r * 128u +
                   ((((uint32_t)ch & 7u) ^ ((uint32_t)r & 7u)) << 4);
  uint32_t hv[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) hv[e] = pack2<kFmt>(v[2 * e], v[2 * e + 1]);
  *reinterpret_cast<uint4*>(dst + o) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
  if (dst_lo)  // the split precisions' low halves
    *reinterpret_cast<uint4*>(dst_lo + o) =
        make_uint4(pack2_low<kFmt>(v[0], v[1], hv[0]), pack2_low<kFmt>(v[2], v[3], hv[1]),
                   pack2_low<kFmt>(v[4], v[5], hv[2]), pack2_low<kFmt>(v[6], v[7], hv[3]));
}
// src_lo (or null): the lo image of a split pair, added in fp32
template <int kFmt>
__global__ void t16_unpack_kernel(const uint8_t* __restrict__ src, int img_cols, float* __restrict__ dst, int ld,
                                  int cols, int64_t m, const uint8_t* __restrict__ src_lo) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m * cols) return;
  const int64_t row = idx / cols;
  const int col = (int)(idx % cols);
  float v = t16_load<kFmt>(src, row, col, img_cols);
  if (src_lo) v += t16_load<kFmt>(src_lo, row, col, img_cols);
  dst[row * ld + col] = v;
}

inline unsigned blocks_of(int64_t n, int per_block) { return (unsigned)((n + per_block - 1) / per_block); }

}  // namespace

size_t t16_image_bytes(int64_t rows, int cols) {
  return (size_t)((rows + 127) / 128) * (size_t)((cols + 63) / 64) * kSlab;
}

cudaError_t launch_t16_pack(const float* src, int ld, int cols, int64_t m, T16Out image, int precision,
                            cudaStream_t st) {
  const int img_cols = (cols + 63) / 64 * 64;
  const int64_t padded = (m + 127) / 128 * 128;
  if (padded == 0) return cudaSuccess;
  LaunchScope scope(kKernIpe, st);  // accounted with the feature kernels (its use in the training step)
  const int vec = (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
  const int64_t total = padded * (img_cols / 8);
  return with_fmt(precision, false, [&](auto fmt, auto) {
    t16_pack_kernel<fmt><<<blocks_of(total, 256), 256, 0, st>>>(src, ld, cols, m, image.hi, img_cols, padded, vec,
                                                                 image.lo);
    return cudaGetLastError();
  });
}

// min_deg = 0, max_deg = 16 (96 features), n = 128 samples per ray: the level kernels' shape
cudaError_t launch_ipe_t16(const float* origins, const float* directions, const float* radii, const float* t,
                           T16Out image, int64_t num_rays, int n, int disable_integration, int precision,
                           cudaStream_t st) {
  if (num_rays == 0) return cudaSuccess;
  if (n != 128) return cudaErrorInvalidValue;
  const int64_t total = num_rays * n * 8;
  return with_fmt(precision, image.lo != nullptr, [&](auto fmt, auto split) {
    LaunchScope scope(kKernIpe, st);
    ipe_t16_kernel<fmt, split><<<blocks_of(total, 256), 256, 0, st>>>(origins, directions, radii, t, image.hi, num_rays,
                                                                       n, disable_integration, image.lo);
    return cudaGetLastError();
  });
}

cudaError_t launch_ipe_points_t16(const float* means, const float* covs, void* image, int64_t num_points,
                                  int disable_integration, int precision, cudaStream_t st) {
  const int64_t padded = (num_points + 127) / 128 * 128;
  if (padded == 0) return cudaSuccess;
  LaunchScope scope(kKernIpe, st);
  const int64_t total = padded * 8;
  return with_fmt(precision, false, [&](auto fmt, auto) {
    ipe_points_t16_kernel<fmt><<<blocks_of(total, 256), 256, 0, st>>>(means, covs, (uint8_t*)image, num_points, padded,
                                                                       disable_integration);
    return cudaGetLastError();
  });
}

cudaError_t launch_t16_unpack(T16 image, int cols, float* dst, int ld, int64_t m, int precision, cudaStream_t st) {
  const int img_cols = (cols + 63) / 64 * 64;
  if (m == 0) return cudaSuccess;
  return with_fmt(precision, false, [&](auto fmt, auto) {
    t16_unpack_kernel<fmt><<<blocks_of(m * cols, 256), 256, 0, st>>>(image.hi, img_cols, dst, ld, cols, m, image.lo);
    return cudaGetLastError();
  });
}

// m rows (a multiple of 128), n in {128, 256}, k in {128, 256}
cudaError_t launch_linear_t16(T16 x, T16 image, T16Out y, int64_t m, int n, int k, const float* r1, const float* r1w,
                              const void* mask, int precision, cudaStream_t st, const void* mask_bits) {
  if (m == 0) return cudaSuccess;
  if (m % 128 != 0 || !(n == 128 || n == 256) || !(k == 128 || k == 256)) return cudaErrorInvalidValue;
  if (mask_bits && (mask || n != 256)) return cudaErrorInvalidValue;
  if (!x.lo != !image.lo || !x.lo != !y.lo) return cudaErrorInvalidValue;  // bf16x3: all three are pairs
  int sms = 0;
  cudaError_t e = num_sms(&sms);
  if (e != cudaSuccess) return e;
  const int slabs = k / 64, halves = n / 128;
  LinearT16Params p{};
  p.x = x.hi, p.image = image.hi, p.y = y.hi;
  p.mask_bits = static_cast<const uint8_t*>(mask_bits);
  p.mask = static_cast<const uint8_t*>(mask), p.r1 = r1, p.r1w = r1w, p.tiles = m / 128, p.n = n, p.k = k;
  if (!x.lo)
    return with_fmt(precision, false, [&](auto fmt, auto) {
      const size_t smem = 1024 + (size_t)slabs * kSlab + linear_tc_image_bytes(n, k) + 128;
      cudaError_t e = allow_smem<linear_t16_kernel<fmt>>(200 * 1024);
      if (e != cudaSuccess) return e;
      const int grid = (int)(p.tiles < sms ? p.tiles : sms);
      LaunchScope scope(kKernLinearTc, st);
      linear_t16_kernel<fmt><<<grid, 256, smem, st>>>(p);
      return cudaGetLastError();
    });
  return with_fmt(precision, true, [&](auto fmt, auto split) {  // bf16x3: linear_t16_x3_kernel
    if constexpr (split) {
      const size_t smem = 1024 + (size_t)(2 * slabs + 4) * kSlab + 64;
      cudaError_t e = allow_smem<linear_t16_x3_kernel<fmt>>((int)(1024 + (size_t)(2 * 4 + 4) * kSlab + 64));
      if (e != cudaSuccess) return e;
      const LinearT16X3Params q{p, x.lo, image.lo, y.lo};
      // a CTA keeps one N-half for good: the grid is a whole number of CTAs per half
      const int64_t per_half = p.tiles < sms / halves ? p.tiles : sms / halves;
      LaunchScope scope(kKernLinearTc, st);
      linear_t16_x3_kernel<fmt><<<(unsigned)(per_half * halves), 288, smem, st>>>(q);
    }
    return cudaGetLastError();
  });
}

cudaError_t launch_color_dgrad_t16(const float* d_rgb, const float* wc, const void* v, T16Out d_v, int64_t m, int k_dim,
                                   int precision, cudaStream_t st) {
  if (m == 0) return cudaSuccess;
  if (k_dim % 64 != 0) return cudaErrorInvalidValue;
  const int64_t total = m * (k_dim / 8);
  return with_fmt(precision, d_v.lo != nullptr, [&](auto fmt, auto split) {
    LaunchScope scope(kKernDgrad, st);
    color_dgrad_t16_kernel<fmt, split><<<blocks_of(total, 256), 256, 0, st>>>(d_rgb, wc, (const uint8_t*)v, d_v.hi, m,
                                                                               k_dim, d_v.lo);
    return cudaGetLastError();
  });
}

// narrow heads: dW[n_dim, k_dim] and db from dy (fp32 [m, n_dim], n_dim = 1 or 3) and a tile-image X; partials +
// fixed-order sum
cudaError_t launch_wgrad_small_n_t16(const float* dy, int n_dim, T16 x, int k_dim, float* part, float* dw, float* db,
                                     int accumulate, int64_t m, int precision, cudaStream_t st, float scale) {
  if (m == 0 || n_dim == 0) return cudaSuccess;
  if (!(n_dim == 1 || n_dim == 3) || !(k_dim == 128 || k_dim == 256)) return cudaErrorInvalidValue;
  int sms = 0;
  cudaError_t e = num_sms(&sms);
  if (e != cudaSuccess) return e;
  int64_t want = 4 * (int64_t)sms;  // four resident blocks per SM, one wave
  if (want > (m + 63) / 64) want = (m + 63) / 64;
  if (want < 1) want = 1;
  const int slices = (int)want;
  const int64_t rows = (m + slices - 1) / slices;
  e = with_fmt(precision, x.lo != nullptr, [&](auto fmt, auto split) {
    LaunchScope scope(kKernWgrad, st);
    if (n_dim == 1)
      wgrad_small_n_t16_kernel<fmt, 1, split><<<slices, 256, 0, st>>>(dy, x.hi, k_dim, part, m, rows, x.lo);
    else
      wgrad_small_n_t16_kernel<fmt, 3, split><<<slices, 256, 0, st>>>(dy, x.hi, k_dim, part, m, rows, x.lo);
    return cudaGetLastError();
  });
  if (e != cudaSuccess) return e;
  return launch_wgrad_reduce(part, slices, n_dim, k_dim, dw, db, accumulate, st, scale);
}

}  // namespace mipnerf
