// linear_tc.cu — a stand-alone wgmma linear layer for the training step's forward and dgrad GEMMs:
//   Y[M, N] = epilogue( X[M, K] . B[N, K]^T ),   N in {128, 256},  K in {96, 128, 256},  fp32 in / fp32 out,
// 16-bit operands (bf16 / fp16) rounded while staging, fp32 accumulation in registers.
//
// The activations of a training step are HBM-bound (M = rays x samples ~ 5e5 rows, every GEMM reads and writes
// ~0.5 GB) while the weights are tiny, so the kernel is organised around the weights:
//   * persistent CTAs (one per SM); the whole B operand (<= 128 KB, pre-swizzled image written by
//     pack_linear_image_kernel) is fetched ONCE per CTA with cp.async.bulk and stays in shared memory;
//   * per 128-row tile: all 256 threads stage the tile of X cooperatively (coalesced float4 loads, 8 in flight per
//     thread, fp32 -> 16-bit, SW128 K-major slabs: the layout and descriptors validated by mipnerf_b200_selftest_umma),
//     then warpgroup g issues the wgmma (M = 64, N = 128, K = 16) of rows 64 g.. and applies the epilogue from its
//     register accumulators straight to global memory:  + bias[col]  + row_bias[row / row_div][col]  + prev[row][col]
//     + r1[row]*r1w[col], ReLU, ReLU-mask by another activation (dgrad).
#include "kernels.h"
#include "mlp_tc.h"
#include "profile.h"
#include "tc_common.cuh"

namespace mipnerf {
namespace {

using namespace tc;

// B[n][k] = w[n * ldw + col0 + k]            (transposed == 0: forward, rows of W, columns col0.. of its input dim)
//         = w[(row0 + k) * ldw + n]          (transposed == 1: dgrad, B = W[row0.., :n_dim]^T)
// written as slabs of [n rows x 128 B] in the 128-byte-swizzle K-major layout, zero padded to whole slabs.
// lo != 0: fl16(v - fl16(v)), the low half of the split precisions
template <int kFmt>
__global__ void pack_linear_image_kernel(const float* __restrict__ w, int ldw, int off, int transposed,
                                         uint8_t* __restrict__ image, int n, int k, int lo) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int slabs = (k + 63) / 64;
  if (idx >= n * slabs * 64) return;
  const int row = idx / (slabs * 64);
  const int kk = idx % (slabs * 64);
  float v = 0.f;
  if (kk < k) v = transposed ? w[(size_t)(off + kk) * ldw + row] : w[(size_t)row * ldw + off + kk];
  if (lo) v -= from16<kFmt>(to16<kFmt>(v));
  uint16_t* dst = reinterpret_cast<uint16_t*>(image + (size_t)(kk / 64) * n * 128 + sw128_offset(row, kk % 64));
  *dst = to16<kFmt>(v);
}

struct LinearTcParams {
  const float* x;        // [M, ldx], the K columns used start at column 0
  int ldx;
  const uint8_t* image;  // packed B
  float* y;              // [M, ldy]
  int ldy;
  int64_t m;
  int n, k;
  const float* bias;      // [n] or null
  const float* row_bias;  // [M / row_div, n] or null (per-ray view-direction term)
  int row_div;
  const float* prev;      // [M, ldy] or null: added before the activation (second K pass of a concatenated input)
  const float* r1;        // [M] or null, with r1w [n]: rank-1 term r1[row] * r1w[col] (density head in dgrad)
  const float* r1w;
  const float* mask;      // [M, ldy] or null: output zeroed where mask <= 0 (ReLU backward)
  int relu;
};

__device__ __forceinline__ void named_bar(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// 256 threads = two warpgroups, persistent over 128-row tiles.  Per tile all threads stage X (fp32 -> 16-bit SW128
// slabs), then warpgroup g runs the wgmma of rows 64 g .. 64 g + 63 over N in 128-column chunks and applies the epilogue
// from its register accumulators straight to global memory.
template <int kFmt>
__global__ void __launch_bounds__(256, 1) linear_tc_kernel(const LinearTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);  // SW128 atoms need 1024-B alignment
  const int slabs = (p.k + 63) / 64;
  uint8_t* sA = smem;
  uint8_t* sB = sA + (size_t)slabs * 16384;
  uint64_t* bar_b = reinterpret_cast<uint64_t*>(sB + (size_t)slabs * p.n * 128);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, wq = warp & 3;
  if (tid == 0) {
    mbar_init(bar_b, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {  // the weights: once per CTA
    mbar_arrive_expect_tx(bar_b, (uint32_t)(slabs * p.n * 128));
    for (int s = 0; s < slabs; ++s)
      bulk_g2s(sB + (size_t)s * p.n * 128, p.image + (size_t)s * p.n * 128, (uint32_t)(p.n * 128), bar_b);
  }
  mbar_wait(bar_b, 0);
  const int64_t tiles = (p.m + 127) / 128;
  const uint32_t a_u = smem_u32(sA) + (uint32_t)wg * 8192u, b_u = smem_u32(sB);
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t row0 = tile * 128;
    for (int s = 0; s < slabs; ++s) {
      float4 f[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {  // 8 coalesced loads in flight per thread before anything else
        const int idx = i * 256 + tid;
        const int r = idx >> 4, k0 = s * 64 + (idx & 15) * 4;
        f[i] = (row0 + r < p.m && k0 < p.k)
                   ? __ldg(reinterpret_cast<const float4*>(p.x + (row0 + r) * (int64_t)p.ldx + k0))
                   : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int idx = i * 256 + tid;
        const int r = idx >> 4, q = idx & 15;
        *reinterpret_cast<uint2*>(sA + (size_t)s * 16384 + sw128_offset(r, (q >> 1) * 8) + (q & 1) * 8) =
            make_uint2(pack2<kFmt>(f[i].x, f[i].y), pack2<kFmt>(f[i].z, f[i].w));
      }
    }
    fence_proxy_async_smem();  // st.shared operand -> async proxy
    __syncthreads();
    const int r_lo = 64 * wg + 16 * wq + (lane >> 2);
    for (int nc = 0; nc < p.n; nc += 128) {
      float acc[64];
      wgmma_fence_acc(acc);
      wgmma_fence();
      uint32_t first = 0;
      for (int s = 0; s < slabs; ++s) {
        const int steps = ((p.k - s * 64) < 64 ? (p.k - s * 64) : 64) / 16;
        for (int j = 0; j < steps; ++j) {
          wgmma_m64n128k16<kFmt>(acc, make_sw128_desc(a_u + (uint32_t)s * 16384u + 32u * j),
                                 make_sw128_desc(b_u + (uint32_t)(s * p.n + nc) * 128u + 32u * j), first);
          first = 1;
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = row0 + r_lo + 8 * h;
        if (row >= p.m) continue;
        const float rv = p.r1 ? __ldg(p.r1 + row) : 0.f;
        float* yr = p.y + row * (int64_t)p.ldy;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = nc + 8 * j + 2 * (lane & 3);
          float o0 = acc[4 * j + 2 * h], o1 = acc[4 * j + 2 * h + 1];
          auto add2 = [&](const float* src) {
            const float2 t = __ldg(reinterpret_cast<const float2*>(src));
            o0 += t.x, o1 += t.y;
          };
          if (p.bias) add2(p.bias + col);
          if (p.row_bias) add2(p.row_bias + (row / p.row_div) * p.n + col);
          if (p.prev) {  // may alias y (in-place second K pass): a plain coherent load, not the read-only path
            const float2 t = *reinterpret_cast<const float2*>(p.prev + row * (int64_t)p.ldy + col);
            o0 += t.x, o1 += t.y;
          }
          if (p.r1) {
            const float2 t = __ldg(reinterpret_cast<const float2*>(p.r1w + col));
            o0 = fmaf(rv, t.x, o0), o1 = fmaf(rv, t.y, o1);
          }
          if (p.relu) o0 = fmaxf(o0, 0.f), o1 = fmaxf(o1, 0.f);
          if (p.mask) {
            const float2 t = __ldg(reinterpret_cast<const float2*>(p.mask + row * (int64_t)p.ldy + col));
            if (!(t.x > 0.f)) o0 = 0.f;
            if (!(t.y > 0.f)) o1 = 0.f;
          }
          *reinterpret_cast<float2*>(yr + col) = make_float2(o0, o1);
        }
      }
    }
    __syncthreads();  // both warpgroups' wgmmas are done with the A slabs before the next tile is staged
  }
}

// ---------------------------------------------------------------------------------------------------------------
// wgrad on the tensor core:  part[s][n][kg] = sum_{m in slice s} dY[m, n] * Xc[m, kg],
//   Xc = [X1 (k1 cols) | X2[m / x2_row_div] (k2 cols)], column K of each partial row = the bias gradient (column sums
//   of dY): the layout wgrad_reduce_kernel expects.
// The reduction index of dW = dY^T . X is the row m, and a row-major [m][col] tile IS the canonical "MN-major" wgmma
// operand (transpose bits of the instruction): 64 consecutive columns (128 B) x 8 rows form one 128-byte-swizzle atom,
// column blocks LBO apart, 8-row groups SBO apart.  Staging is therefore a straight copy: a warp reads one whole row
// (1 KB, coalesced), rounds to 16 bit and stores one 16-byte chunk per lane at the swizzled position of the same row.
//   grid (slices, 128-column k tiles); one CTA per SM covers ALL n_dim <= 256 output rows (warpgroup g: rows 128 g..,
//   two M = 64 register accumulators), so dY is read once per k tile;
//   warps 0-7 stage 64-row slabs into a 3-deep ring (tile-image operands arrive by bulk copy from warp 8), then run
//   4 K-steps of wgmma per slab and free the stage (one arrive per warpgroup); after the last slab they write the
//   partial rows from the accumulators and add up the bias gradient (column sums of dY, kept in fp32 by the thread
//   that staged the column) in a fixed order.
// ---------------------------------------------------------------------------------------------------------------
struct WgradTcParams {
  const float* dy;  // [M, n_dim]
  int n_dim;
  const float* x1;  // [M, ld1]
  int ld1, k1;
  const float* x2;  // [M / x2_row_div, ld2] or null
  int ld2, k2, x2_row_div;
  float* part;      // [slices, n_dim, K + 1]
  int64_t m, slice_rows;
  // dy / x1 / x2 are 16-bit tile images (train_t16.cu) instead of fp32 row-major matrices; x1's / x2's image has
  // ceil(k / 64) slabs per tile (x2 as an image: x2_row_div == 1).
  int dy_t16, x1_t16, x2_t16;
  // optional by-product when x1 is a 256-column tile image: its sign mask, [m][32 bytes], bit c of a row = x1[row][c] > 0.
  // The dgrad GEMM that follows needs exactly this (the ReLU mask of the layer input) and then reads 32 bytes per row
  // instead of the 512-byte activation row again.
  uint8_t* mask_out;
  // bf16x3: the lo images of the tile-image operands (dy, x1 and x2 when they are images); fp32 operands are split
  // while staging.
  const uint8_t *dy_lo, *x1_lo, *x2_lo;
};

constexpr int kWgStages = 3;
constexpr int kWgSlab = 64;                    // rows (reduction steps) per stage
constexpr uint32_t kWgOperand = kWgSlab * 512; // 64 rows x 256 cols x 2 B
constexpr uint32_t kWgStage = 2 * kWgOperand;
constexpr uint32_t kWgBlock = kWgSlab * 128;   // one 64-column block of a slab
constexpr int kWgK = 128;                      // output columns per CTA (the wgmma N)
// bf16x3 keeps the three 64 KB stages and halves the slab instead: 32 rows of dY hi, X hi, dY lo and X lo per stage
// (4 x 16 KB), so the ring stays 192 KB and as deep; the partial sums are added in the same fixed order either way.
constexpr int kWgSlabX3 = 32;
static_assert(4 * kWgSlabX3 * 512 == kWgStage, "a bf16x3 stage is as large as a 16-bit one");

template <int kFmt>
__device__ __forceinline__ float2 unpack16x2(uint32_t v) {
  if (kFmt == 1) return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&v));
  return __half22float2(*reinterpret_cast<__half2*>(&v));
}

// eight fp32 values as hi = fl16(x) and lo = fl16(x - hi), 16 bytes each
template <int kFmt>
__device__ __forceinline__ void stage8_split(uint8_t* hi, uint8_t* lo, const float4 (&f)[2]) {
  const float v[8] = {f[0].x, f[0].y, f[0].z, f[0].w, f[1].x, f[1].y, f[1].z, f[1].w};
  uint32_t h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    h[e] = pack2<kFmt>(v[2 * e], v[2 * e + 1]);
    l[e] = pack2_low<kFmt>(v[2 * e], v[2 * e + 1], h[e]);
  }
  *reinterpret_cast<uint4*>(hi) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo) = make_uint4(l[0], l[1], l[2], l[3]);
}

template <int kFmt, bool kX3 = false>
__global__ void __launch_bounds__(288, 1) wgrad_mn_kernel(const WgradTcParams p) {
  // rows per slab, and the operand / 64-column block sizes of a slab; kX3 adds the lo operands kLo bytes behind the hi
  // ones in the stage: [dY hi][X hi][dY lo][X lo]
  constexpr int kWgSlab = kX3 ? kWgSlabX3 : ::mipnerf::kWgSlab;
  constexpr uint32_t kWgOperand = kWgSlab * 512, kWgBlock = kWgSlab * 128, kLo = 2 * kWgOperand;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* ring = smem;
  float* bias_s = reinterpret_cast<float*>(ring + kWgStages * kWgStage);  // [8 warps][256]
  uint64_t* bars = reinterpret_cast<uint64_t*>(bias_s + 8 * 256);
  uint64_t* full = bars;                  // [stages], 8 arrivals (one per stager warp) (+ 1 with tx bytes)
  uint64_t* empty = bars + kWgStages;     // [stages], one arrival per warpgroup once its wgmmas have read the stage
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = p.k1 + p.k2;
  const int kg0 = blockIdx.y * kWgK;
  const int nk = K - kg0 < kWgK ? K - kg0 : kWgK;  // valid output columns of this k tile
  const int nk_mma = (nk + 63) & ~63;            // whole 64-column blocks (padding staged as zeros)
  const int n_halves = p.n_dim >> 7;
  const int64_t m_begin = (int64_t)blockIdx.x * p.slice_rows;
  const int64_t m_end = (m_begin + p.slice_rows) < p.m ? (m_begin + p.slice_rows) : p.m;
  const bool has_rows = m_begin < m_end;
  const int slabs = has_rows ? (int)((m_end - m_begin + kWgSlab - 1) / kWgSlab) : 0;
  // the k tile lies in X1 or in X2 (the launcher guarantees it never straddles)
  const bool in_x1 = kg0 < p.k1;
  const float* xs = in_x1 ? p.x1 : p.x2;
  const int ldx = in_x1 ? p.ld1 : p.ld2, xdiv = in_x1 ? 1 : p.x2_row_div, xc0 = in_x1 ? kg0 : kg0 - p.k1;
  const bool xvec = (ldx & 3) == 0 && xdiv == 1 && (xc0 & 3) == 0 && (nk & 7) == 0 &&
                    (reinterpret_cast<uintptr_t>(xs) & 15) == 0;
  // tile-image operands arrive by bulk copy (warp 9), fp32 operands through the stager warps' registers
  const bool a16 = p.dy_t16 != 0, b16 = in_x1 ? p.x1_t16 != 0 : p.x2_t16 != 0;
  // fp32 operand whose row index is the same for a whole 64-row slab (the per-ray view encodings, one ray = 128 rows):
  // fetched once per slab instead of once per row
  const bool x_per_slab = !b16 && !xvec && (xdiv & 63) == 0;
  const bool bias_read = a16 && blockIdx.y == 0;  // column sums of dY are then taken from the staged tile
  // the 256-column sign mask is split between the two k tiles of x1: lanes [mlane0, mlane0 + 16) write their bytes
  const bool mask_write = p.mask_out != nullptr && b16 && in_x1 && kg0 < 256 && nk == kWgK;
  const int mlane0 = kg0 >> 3;
  const bool reader = bias_read || mask_write;    // the stager warps read staged tile images out of shared memory
  const int a_blocks = p.n_dim >> 6, b_blocks = nk_mma >> 6;

  if (tid == 0) {
    for (int s = 0; s < kWgStages; ++s) {
      mbar_init(&full[s], ((a16 && b16) ? 0 : 8) + ((a16 || b16) ? 1 : 0));
      mbar_init(&empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ============================== bulk producer (tile-image operands) ==============================
    if (lane == 0 && (a16 || b16)) {
      const uint8_t* dy16 = reinterpret_cast<const uint8_t*>(p.dy);
      const uint8_t* x16 = reinterpret_cast<const uint8_t*>(in_x1 ? p.x1 : p.x2);
      const uint8_t* x16_lo = in_x1 ? p.x1_lo : p.x2_lo;
      const int x_slabs = ((in_x1 ? p.k1 : p.k2) + 63) >> 6;
      const uint32_t bytes = (uint32_t)((a16 ? a_blocks : 0) + (b16 ? b_blocks : 0)) * kWgBlock * (kX3 ? 2u : 1u);
      // the operand tiles stream through once (0.5 GB per launch): evict-first, so that the 39 MB of partial sums this
      // launch writes are still in L2 when the reduction kernel reads them
      const uint64_t stream_policy = l2_policy_evict_first();
      for (int it = 0; it < slabs; ++it) {
        const int s = it % kWgStages;
        if (it >= kWgStages) mbar_wait(&empty[s], (uint32_t)(it / kWgStages - 1) & 1u);
        uint8_t* sa = ring + (size_t)s * kWgStage;
        uint8_t* sb = sa + kWgOperand;
        const int64_t row0 = m_begin + (int64_t)it * kWgSlab;  // a multiple of the slab: a part of a 128-row tile
        const size_t tile = (size_t)(row0 >> 7), half = (size_t)(row0 & 127) * 128;
        mbar_arrive_expect_tx(&full[s], bytes);
        if (a16)
          for (int b = 0; b < a_blocks; ++b) {
            const size_t o = (tile * a_blocks + b) * 16384 + half;
            bulk_g2s_hint(sa + (size_t)b * kWgBlock, dy16 + o, kWgBlock, &full[s], stream_policy);
            if (kX3) bulk_g2s_hint(sa + kLo + (size_t)b * kWgBlock, p.dy_lo + o, kWgBlock, &full[s], stream_policy);
          }
        if (b16)
          for (int b = 0; b < b_blocks; ++b) {
            const size_t o = (tile * x_slabs + (xc0 >> 6) + b) * 16384 + half;
            bulk_g2s_hint(sb + (size_t)b * kWgBlock, x16 + o, kWgBlock, &full[s], stream_policy);
            if (kX3) bulk_g2s_hint(sb + kLo + (size_t)b * kWgBlock, x16_lo + o, kWgBlock, &full[s], stream_policy);
          }
      }
    }
  } else {
    // ========================= stagers = wgmma warpgroups (warpgroup g: output rows 128 g ..) =========================
    // Both operands are MN-major (the reduction index m is the row of the staged tiles): 64 consecutive columns (128 B)
    // x 8 rows form one 128-byte-swizzle atom, 64-column blocks kWgBlock apart (leading offset), 8-row groups 1 KB
    // apart (stride offset).  Accumulators: rows 128 g + 64 b .. of the [n_dim x 128] partial, b = 0, 1.
    const int wg = warp >> 2, wq = warp & 3;
    const bool mma_on = wg < n_halves;
    float acc0[64], acc1[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc0[i] = 0.f, acc1[i] = 0.f;
    float bs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // column sums of dY, columns lane*8 .. +7, this warp's rows
    const int c8 = lane * 8;
    const bool a_on = c8 < p.n_dim, b_on = c8 < nk_mma;
    const uint32_t blk = (uint32_t)(lane >> 3) * kWgBlock, chunk = (uint32_t)(lane & 7);
    for (int it = 0; it < slabs; ++it) {
      const int s = it % kWgStages;
      uint8_t* sa = ring + (size_t)s * kWgStage;
      uint8_t* sb = sa + kWgOperand;
      if (!(a16 && b16)) {
      if (it >= kWgStages) mbar_wait(&empty[s], (uint32_t)(it / kWgStages - 1) & 1u);
      const int64_t m0 = m_begin + (int64_t)it * kWgSlab;
      float4 xs0 = make_float4(0.f, 0.f, 0.f, 0.f), xs1 = xs0;
      if (x_per_slab && c8 < nk) {
        const float* src = xs + (m0 / xdiv) * (int64_t)ldx + xc0 + c8;
        float t[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) t[e] = (c8 + e < nk) ? __ldg(src + e) : 0.f;
        xs0 = make_float4(t[0], t[1], t[2], t[3]), xs1 = make_float4(t[4], t[5], t[6], t[7]);
      }
#pragma unroll
      for (int half = 0; half < kWgSlab / 32; ++half) {
        float4 fa[4][2], fb[4][2];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = warp + 8 * (half * 4 + i);
          const int64_t row = m0 + r;
          const bool ok = row < m_end;
          fa[i][0] = fa[i][1] = fb[i][0] = fb[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok && a_on && !a16) {
            const float4* src = reinterpret_cast<const float4*>(p.dy + row * (int64_t)p.n_dim + c8);
            fa[i][0] = __ldg(src), fa[i][1] = __ldg(src + 1);
          }
          if (ok && c8 < nk && !b16) {
            if (x_per_slab) {
              fb[i][0] = xs0, fb[i][1] = xs1;
            } else if (xvec) {
              const float4* src = reinterpret_cast<const float4*>(xs + row * (int64_t)ldx + xc0 + c8);
              fb[i][0] = __ldg(src), fb[i][1] = __ldg(src + 1);
            } else {
              const float* src = xs + (row / xdiv) * (int64_t)ldx + xc0 + c8;
              float t[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) t[e] = (c8 + e < nk) ? __ldg(src + e) : 0.f;
              fb[i][0] = make_float4(t[0], t[1], t[2], t[3]), fb[i][1] = make_float4(t[4], t[5], t[6], t[7]);
            }
          }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = warp + 8 * (half * 4 + i);
          const uint32_t off = blk + (uint32_t)r * 128u + ((chunk ^ (uint32_t)(r & 7)) << 4);
          if (a_on && !a16) {
            bs[0] += fa[i][0].x, bs[1] += fa[i][0].y, bs[2] += fa[i][0].z, bs[3] += fa[i][0].w;
            bs[4] += fa[i][1].x, bs[5] += fa[i][1].y, bs[6] += fa[i][1].z, bs[7] += fa[i][1].w;
            if constexpr (kX3) {
              stage8_split<kFmt>(sa + off, sa + kLo + off, fa[i]);
            } else {
            *reinterpret_cast<uint4*>(sa + off) =
                make_uint4(pack2<kFmt>(fa[i][0].x, fa[i][0].y), pack2<kFmt>(fa[i][0].z, fa[i][0].w),
                           pack2<kFmt>(fa[i][1].x, fa[i][1].y), pack2<kFmt>(fa[i][1].z, fa[i][1].w));
            }
          }
          if (b_on && !b16) {
            if constexpr (kX3) {
              stage8_split<kFmt>(sb + off, sb + kLo + off, fb[i]);
            } else {
            *reinterpret_cast<uint4*>(sb + off) =
                make_uint4(pack2<kFmt>(fb[i][0].x, fb[i][0].y), pack2<kFmt>(fb[i][0].z, fb[i][0].w),
                           pack2<kFmt>(fb[i][1].x, fb[i][1].y), pack2<kFmt>(fb[i][1].z, fb[i][1].w));
            }
          }
        }
      }
      fence_proxy_async_smem();  // this thread's st.shared -> visible to the tensor core's (async-proxy) reads
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[s]);
      }
      mbar_wait(&full[s], (uint32_t)(it / kWgStages) & 1u);
      if (mma_on) {
        const uint32_t sa_u = smem_u32(sa), sb_u = smem_u32(sb);
        wgmma_fence_acc(acc0);
        wgmma_fence_acc(acc1);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < kWgSlab / 16; ++j) {  // 16 rows = two 8-row groups = 2 KB further into every block
          const uint64_t bd = gmma_desc(sb_u + j * 2048, kWgBlock, 1024, 1);
          const uint64_t ad0 = gmma_desc(sa_u + (2 * wg) * kWgBlock + j * 2048, kWgBlock, 1024, 1);
          const uint64_t ad1 = gmma_desc(sa_u + (2 * wg + 1) * kWgBlock + j * 2048, kWgBlock, 1024, 1);
          wgmma_m64n128k16<kFmt, 1, 1>(acc0, ad0, bd, 1u);
          if (kX3) {  // dY_lo . X_hi + dY_hi . X_lo, the level kernel's order
            wgmma_m64n128k16<kFmt, 1, 1>(acc0, ad0 + kLo / 16, bd, 1u);
            wgmma_m64n128k16<kFmt, 1, 1>(acc0, ad0, bd + kLo / 16, 1u);
          }
          wgmma_m64n128k16<kFmt, 1, 1>(acc1, ad1, bd, 1u);
          if (kX3) {
            wgmma_m64n128k16<kFmt, 1, 1>(acc1, ad1 + kLo / 16, bd, 1u);
            wgmma_m64n128k16<kFmt, 1, 1>(acc1, ad1, bd + kLo / 16, 1u);
          }
        }
        wgmma_commit();
      }
      if (reader) {  // operands that arrived as tile images: column sums of dY, sign mask of X, from shared memory
        if (mask_write && lane >= mlane0 && lane < mlane0 + 16) {
          const uint32_t mblk = (uint32_t)((lane - mlane0) >> 3) * kWgBlock;
          const int64_t m0r = m_begin + (int64_t)it * kWgSlab;
#pragma unroll
          for (int i = 0; i < kWgSlab / 8; ++i) {
            const int r = warp + 8 * i;
            const uint4 w = *reinterpret_cast<const uint4*>(sb + mblk + (uint32_t)r * 128u + ((chunk ^ (uint32_t)(r & 7)) << 4));
            const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
            uint32_t bits = 0;
#pragma unroll
            for (int e = 0; e < 4; ++e) {  // a 16-bit float is > 0 iff its bits, read as a signed integer, are > 0
              bits |= ((int16_t)(ww[e] & 0xffffu) > 0 ? 1u : 0u) << (2 * e);
              bits |= ((int32_t)ww[e] >= 0x00010000 ? 1u : 0u) << (2 * e + 1);
            }
            p.mask_out[(m0r + r) * 32 + lane] = (uint8_t)bits;  // byte = columns lane*8 .. +7: 32 B per row, coalesced
          }
        }
        if (bias_read && a_on) {
#pragma unroll
          for (int i = 0; i < kWgSlab / 8; ++i) {
            const int r = warp + 8 * i;
            const uint32_t o = blk + (uint32_t)r * 128u + ((chunk ^ (uint32_t)(r & 7)) << 4);
            const uint4 w = *reinterpret_cast<const uint4*>(sa + o);
            float2 f0 = unpack16x2<kFmt>(w.x), f1 = unpack16x2<kFmt>(w.y), f2 = unpack16x2<kFmt>(w.z),
                   f3 = unpack16x2<kFmt>(w.w);
            if (kX3) {  // dY = hi + lo
              const uint4 wl = *reinterpret_cast<const uint4*>(sa + kLo + o);
              const float2 l0 = unpack16x2<kFmt>(wl.x), l1 = unpack16x2<kFmt>(wl.y), l2 = unpack16x2<kFmt>(wl.z),
                           l3 = unpack16x2<kFmt>(wl.w);
              f0.x += l0.x, f0.y += l0.y, f1.x += l1.x, f1.y += l1.y;
              f2.x += l2.x, f2.y += l2.y, f3.x += l3.x, f3.y += l3.y;
            }
            bs[0] += f0.x, bs[1] += f0.y, bs[2] += f1.x, bs[3] += f1.y;
            bs[4] += f2.x, bs[5] += f2.y, bs[6] += f3.x, bs[7] += f3.y;
          }
        }
      }
      if (mma_on) {
        wgmma_wait<0>();
        wgmma_fence_acc(acc0);
        wgmma_fence_acc(acc1);
      }
      named_bar(2 + wg, 128);  // the warpgroup's wgmmas and readers are done with the stage
      if ((tid & 127) == 0) mbar_arrive(&empty[s]);
    }
    // ---- bias gradient: per-warp column sums -> fixed-order sum over the 8 warps
    if (a_on) {
#pragma unroll
      for (int e = 0; e < 8; ++e) bias_s[warp * 256 + c8 + e] = bs[e];
    }
    named_bar(1, 256);
    float* out = p.part + (size_t)blockIdx.x * p.n_dim * (K + 1);
    if (blockIdx.y == 0 && tid < p.n_dim) {
      float t = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) t += bias_s[w8 * 256 + tid];
      out[(size_t)tid * (K + 1) + K] = t;
    }
    // ---- accumulators -> partial rows
    if (mma_on) {
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int nr = 128 * wg + 64 * b + 16 * wq + (lane >> 2) + 8 * h;
          float* orow = out + (size_t)nr * (K + 1) + kg0;
#pragma unroll
          for (int jj = 0; jj < 16; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * jj + 2 * (lane & 3) + e;
              if (c < nk) orow[c] = b ? acc1[4 * jj + 2 * h + e] : acc0[4 * jj + 2 * h + e];
            }
        }
    }
  }
}

}  // namespace

size_t linear_tc_image_bytes(int n, int k) { return (size_t)((k + 63) / 64) * n * 128; }

bool linear_tc_shape_ok(int n, int k) { return (n == 128 || n == 256) && (k == 96 || k == 128 || k == 256); }

cudaError_t launch_pack_linear_image(const float* w, int ldw, int off, int transposed, void* image, int n, int k,
                                     int precision, cudaStream_t st, int lo) {
  const int total = n * ((k + 63) / 64) * 64;
  LaunchScope scope(kKernPackWeights, st);
  return with_fmt(precision, false, [&](auto fmt, auto) {
    pack_linear_image_kernel<fmt><<<(total + 255) / 256, 256, 0, st>>>(w, ldw, off, transposed, (uint8_t*)image, n, k,
                                                                       lo);
    return cudaGetLastError();
  });
}

// precision: MIPNERF_B200_BF16 / _FP16
cudaError_t launch_linear_tc(const float* x, int ldx, const void* image, float* y, int ldy, int64_t m, int n, int k,
                             const float* bias, const float* row_bias, int row_div, const float* prev,
                             const float* r1, const float* r1w, const float* mask, int relu, int precision,
                             cudaStream_t st) {
  if (m == 0) return cudaSuccess;
  if (!linear_tc_shape_ok(n, k) || ldx % 4 != 0 || ldy % 4 != 0) return cudaErrorInvalidValue;
  int sms = 0;
  cudaError_t e = num_sms(&sms);
  if (e != cudaSuccess) return e;
  const int slabs = (k + 63) / 64;
  const size_t smem = 1024 + (size_t)slabs * 16384 + linear_tc_image_bytes(n, k) + 64;
  LinearTcParams p{};
  p.x = x, p.ldx = ldx, p.image = static_cast<const uint8_t*>(image), p.y = y, p.ldy = ldy, p.m = m, p.n = n, p.k = k;
  p.bias = bias, p.row_bias = row_bias, p.row_div = row_div < 1 ? 1 : row_div, p.prev = prev;
  p.r1 = r1, p.r1w = r1w, p.mask = mask, p.relu = relu;
  const int64_t tiles = (m + 127) / 128;
  const int grid = (int)(tiles < sms ? tiles : sms);
  return with_fmt(precision, false, [&](auto fmt, auto) {
    cudaError_t e = allow_smem<linear_tc_kernel<fmt>>(200 * 1024);
    if (e != cudaSuccess) return e;
    LaunchScope scope(kKernLinearTc, st);
    linear_tc_kernel<fmt><<<grid, 256, smem, st>>>(p);
    return cudaGetLastError();
  });
}

bool wgrad_tc_shape_ok(int n_dim) { return n_dim == 128 || n_dim == 256; }

cudaError_t launch_wgrad_mn_partials(const WgradOperand& dy, int n_dim, const WgradOperand& x1, int k1,
                                     const WgradOperand& x2_in, int k2, int x2_row_div, float* part, int64_t m,
                                     int max_slices, int precision, int* slices_out, cudaStream_t st,
                                     void* mask_out) {
  const WgradOperand& x2 = x2_in.absent() ? x1 : x2_in;  // no x2: x1 again, with no columns
  if (x2_in.absent()) k2 = 0;
  // bf16x3 when dy is a pair; then x1 and an image x2 are pairs too, and otherwise no operand has a lo image
  auto paired = [](const WgradOperand& o) { return o.is_image() && o.image.lo != nullptr; };
  const bool x3 = paired(dy);
  if (paired(x1) != x3 || (x2.is_image() && k2 > 0 && paired(x2) != x3)) return cudaErrorInvalidValue;
  if (x2_row_div < 1) x2_row_div = 1;
  const int K = k1 + k2;
  if (!(k2 == 0 || k1 % 256 == 0) || !(n_dim == 128 || n_dim == 256)) return cudaErrorInvalidValue;
  if (dy.f32 && dy.ld != n_dim) return cudaErrorInvalidValue;
  if ((dy.is_image() || x1.is_image() || x2.is_image()) && m % 128 != 0) return cudaErrorInvalidValue;
  if (x2.is_image() && k2 > 0 && x2_row_div != 1) return cudaErrorInvalidValue;
  int sms = 0;
  cudaError_t e = num_sms(&sms);
  if (e != cudaSuccess) return e;
  const int k_tiles = (K + kWgK - 1) / kWgK;
  int64_t slices = sms / k_tiles;  // one CTA per SM, one wave
  const int slab = x3 ? kWgSlabX3 : kWgSlab;
  const int64_t by_rows = (m + slab - 1) / slab;
  if (slices > by_rows) slices = by_rows;
  if (slices > max_slices) slices = max_slices;
  if (slices < 1) slices = 1;
  int64_t slice_rows = (m + slices - 1) / slices;
  slice_rows = (slice_rows + slab - 1) / slab * slab;
  const size_t smem = 1024 + (size_t)kWgStages * kWgStage + 8 * 256 * sizeof(float) + 128;
  auto data = [](const WgradOperand& o) { return o.is_image() ? reinterpret_cast<const float*>(o.image.hi) : o.f32; };
  WgradTcParams p{};
  p.dy = data(dy), p.n_dim = n_dim, p.x1 = data(x1), p.ld1 = x1.ld, p.k1 = k1;
  p.x2 = data(x2), p.ld2 = x2.ld, p.k2 = k2, p.x2_row_div = x2_row_div, p.part = part, p.m = m;
  p.slice_rows = slice_rows, p.dy_t16 = dy.is_image(), p.x1_t16 = x1.is_image(), p.x2_t16 = x2.is_image();
  p.mask_out = (x1.is_image() && k1 == 256) ? static_cast<uint8_t*>(mask_out) : nullptr;
  p.dy_lo = dy.image.lo, p.x1_lo = x1.image.lo, p.x2_lo = x2.image.lo;
  const dim3 grid((unsigned)slices, (unsigned)k_tiles);
  *slices_out = (int)slices;
  return with_fmt(precision, x3, [&](auto fmt, auto split) {
    cudaError_t e = allow_smem<wgrad_mn_kernel<fmt, split>>((int)smem);
    if (e != cudaSuccess) return e;
    LaunchScope scope(kKernWgradTc, st);
    wgrad_mn_kernel<fmt, split><<<grid, 288, smem, st>>>(p);
    return cudaGetLastError();
  });
}

}  // namespace mipnerf
