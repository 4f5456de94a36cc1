// tc_common.cuh — hand-written sm_90a primitives used by the tensor-core kernels:
// mbarrier, 1-D bulk async copy (TMA engine), wgmma (warpgroup MMA) issue / commit / wait,
// wgmma shared-memory descriptors, and the 128-byte-swizzle K-major operand layout.
//
// Operand layout ("SW128 K-major slab"): rows of 128 bytes (64 16-bit elements along K), 8-row
// swizzle atoms of 1024 bytes, 16-byte chunk index XOR (row & 7).  One slab covers 64 elements of
// K for all rows of the operand; a K extent > 64 uses several slabs.  The same byte-offset
// function is used by (a) the epilogue threads that write the next layer's A operand with
// st.shared, (b) the weight packer that pre-swizzles B in global memory so that a stage load is
// one contiguous cp.async.bulk, and (c) the wgmma descriptor (128-byte swizzle, stride offset
// 1024 B, start address advanced by 32 B per K=16 step).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mipnerf {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- operand layout ---------------------------------------------------------------------------
// byte offset of 16-bit element (row r, k in [0,64)) inside a SW128 K-major slab
__host__ __device__ __forceinline__ uint32_t sw128_offset(int r, int k) {
  return (uint32_t)(r * 128 + ((((k >> 3) ^ (r & 7)) << 4) | ((k & 7) << 1)));
}

// 64-byte-swizzle variant for a 32-element K tail: rows of 64 bytes, 8-row atoms of 512 bytes,
// 16-byte chunk index XOR ((row >> 1) & 3)  (cute Swizzle<2,4,3>).
__host__ __device__ __forceinline__ uint32_t sw64_offset(int r, int k) {
  return (uint32_t)(r * 64 + ((((k >> 3) ^ ((r >> 1) & 3)) << 4) | ((k & 7) << 1)));
}

// 32-byte swizzle, K-major: a [rows x 16 elements] block with rows of 32 bytes, 8-row atoms of 256 bytes, 16-byte chunk
// index XOR ((row >> 2) & 1)  (cute Swizzle<1,4,3>).  One K = 16 MMA reads exactly one such block, and the block is DENSE
// in shared memory (128 rows = 4 KB = 32 lines of 128 B) — with the 128-byte-swizzle layout the same K = 16 slice is 32 B
// out of every one of 128 lines, i.e. four times the shared-memory port time per MMA.
__host__ __device__ __forceinline__ uint32_t sw32_offset(int r, int k) {
  return (uint32_t)(r * 32 + (((((k >> 3) & 1) ^ ((r >> 2) & 1)) << 4) | ((k & 7) << 1)));
}

// ---- mbarrier -----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// MIPNERF_TC_WAIT_HINT_NS: suspend-time hint of mbarrier.try_wait (how long the hardware may park the waiting
// thread before the instruction returns false).  0 = no operand, the implementation's default time limit.
#ifndef MIPNERF_TC_WAIT_HINT_NS
#define MIPNERF_TC_WAIT_HINT_NS 0
#endif
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
#if MIPNERF_TC_WAIT_HINT_NS > 0
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"((uint32_t)MIPNERF_TC_WAIT_HINT_NS)
      : "memory");
#else
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
#endif
  return ok != 0;
}
// Bounded spin: a protocol bug turns into a trap (reported as a launch failure) instead of a hang
// that would wedge the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// ---- async-proxy fences & bulk copy -----------------------------------------------------------------
// generic-proxy st.shared -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// shared -> global 1-D bulk copy (one bulk async-group per call); the issuing thread waits with the two helpers below
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n\tcp.async.bulk.commit_group;" ::"l"(gdst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_store_wait_read() {  // the source may be overwritten
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void bulk_store_wait_all() {  // the writes are complete
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
// L2 eviction policies for the bulk copies of a kernel that streams gigabytes out next to a small, hot working set
// (the training forward: 2.5 GB of activation tiles against a 1.3 MB weight image that every CTA re-reads per ray)
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_s2g_hint(void* gdst, const void* smem_src, uint32_t bytes, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;\n\tcp.async.bulk.commit_group;" ::"l"(
          gdst),
      "r"(smem_u32(smem_src)), "r"(bytes), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void st_global_v4_hint(void* gdst, uint4 v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(gdst), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w), "l"(policy));
}
__device__ __forceinline__ void st_global_v2_hint(float* gdst, float x, float y, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(gdst), "f"(x), "f"(y), "l"(policy));
}
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar,
                                              uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
// global -> shared 1-D bulk copy on the TMA engine, completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA) --------------------------------------------------------------------
// Shared-memory matrix descriptor (PTX "matrix descriptor", sm_90): start >> 4 [0,14), leading byte offset >> 4 [16,30),
// stride byte offset >> 4 [32,46), swizzle mode [62,64) (1 = 128 B, 2 = 64 B, 3 = 32 B).  For the K-major swizzled
// layouts the leading offset is unused and the stride offset is the distance between 8-row groups; a K = 16 step inside
// a swizzle row is +32 B on the start address.  For MN-major operands (wgrad) the leading offset is the distance between
// 64-element MN blocks and the stride offset the distance between 8-row K groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo, uint32_t swizzle) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32) |
         ((uint64_t)swizzle << 62);
}
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t saddr) { return gmma_desc(saddr, 16, 1024, 1); }
__device__ __forceinline__ uint64_t make_sw64_desc(uint32_t saddr) { return gmma_desc(saddr, 16, 512, 2); }
__device__ __forceinline__ uint64_t make_sw32_desc(uint32_t saddr) { return gmma_desc(saddr, 16, 256, 3); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of an accumulator across wgmma issue / wait
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, both operands in shared memory, fp32 accumulate in registers; issued by a
// whole warpgroup.  kFmt: 0 fp16, 1 bf16 operands; kTA / kTB: operand MN-major (transposed) instead of K-major.
// Accumulator fragment of thread t (warp w = t / 32 % 4, lane l): d[4 j + e] = D[16 w + l / 4 + 8 (e / 2)][8 j + 2 (l % 4) + e % 2].
#define MIPNERF_WGMMA_D4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define MIPNERF_WGMMA_D16(i) MIPNERF_WGMMA_D4(i), MIPNERF_WGMMA_D4(i + 4), MIPNERF_WGMMA_D4(i + 8), MIPNERF_WGMMA_D4(i + 12)
#define MIPNERF_WGMMA_M64N128K16(TY)                                                                        \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                        \
               "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "                          \
               "%64, %65, p, 1, 1, %67, %68;\n\t}"                                                          \
               : MIPNERF_WGMMA_D16(0), MIPNERF_WGMMA_D16(16), MIPNERF_WGMMA_D16(32), MIPNERF_WGMMA_D16(48)       \
               : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTA), "n"(kTB))
template <int kFmt, int kTA = 0, int kTB = 0>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if (kFmt == 1) MIPNERF_WGMMA_M64N128K16("bf16");
  else MIPNERF_WGMMA_M64N128K16("f16");
}
// The same with A from REGISTERS (RS form): a[0..3] = this thread's packed 16-bit pairs of the [64 x 16] A tile, in the
// accumulator-fragment positions (rows r, r + 8 with r = 16 w + l / 4; columns 2 (l % 4) and 8 + 2 (l % 4)): a[0] = (r, c),
// a[1] = (r + 8, c), a[2] = (r, c + 8), a[3] = (r + 8, c + 8).  The registers must not change until the wgmma completed.
#define MIPNERF_WGMMA_M64N128K16_RS(TY)                                                                     \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"                                        \
               "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "                          \
               "{%64, %65, %66, %67}, %68, p, 1, 1, %70;\n\t}"                                            \
               : MIPNERF_WGMMA_D16(0), MIPNERF_WGMMA_D16(16), MIPNERF_WGMMA_D16(32), MIPNERF_WGMMA_D16(48)       \
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate), "n"(kTB))
template <int kFmt, int kTB = 0>
__device__ __forceinline__ void wgmma_m64n128k16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc,
                                                    uint32_t accumulate) {
  if (kFmt == 1) MIPNERF_WGMMA_M64N128K16_RS("bf16");
  else MIPNERF_WGMMA_M64N128K16_RS("f16");
}

// ---- fp32 pair arithmetic (two IEEE fp32 operations; kept as helpers so the epilogues read as pairs) ----------------
__device__ __forceinline__ void fadd2(float& a, float& b, float ca, float cb) {
  a = __fadd_rn(a, ca);
  b = __fadd_rn(b, cb);
}
// (acc_a, acc_b) += (xa, xb) * (wa, wb)
__device__ __forceinline__ void ffma2(float& acc_a, float& acc_b, float xa, float xb, float wa, float wb) {
  acc_a = __fmaf_rn(xa, wa, acc_a);
  acc_b = __fmaf_rn(xb, wb, acc_b);
}

// ---- 16-bit operand conversion (kFmt: 0 = fp16, 1 = bf16), low half = first element ---------------------
template <int kFmt>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  if (kFmt == 1) {
    __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&b);
  } else {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}
// same with ReLU fused into the conversion (cvt.rn.relu.*x2.f32): max(x,0) then round
template <int kFmt>
__device__ __forceinline__ uint32_t pack2_relu(float lo, float hi) {
  uint32_t d;
  if (kFmt == 1) asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  else asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
template <int kFmt>
__host__ __device__ __forceinline__ uint16_t to16(float x) {
  if (kFmt == 1) {
    __nv_bfloat16 b = __float2bfloat16_rn(x);
    return *reinterpret_cast<uint16_t*>(&b);
  } else {
    __half h = __float2half_rn(x);
    return *reinterpret_cast<uint16_t*>(&h);
  }
}
template <int kFmt>
__device__ __forceinline__ float from16(uint16_t h) {
  if (kFmt == 1) return __bfloat162float(*reinterpret_cast<__nv_bfloat16*>(&h));
  return __half2float(*reinterpret_cast<__half*>(&h));
}
// The low halves of a pair whose high halves are `hi` = pack2(lo_el, hi_el): fl16(x - fl16(x)), the second operand of the
// split ("x3") precisions, as the level kernel rounds it
template <int kFmt>
__device__ __forceinline__ uint32_t pack2_low(float a, float b, uint32_t hi) {
  const float fa = from16<kFmt>((uint16_t)(hi & 0xffffu)), fb = from16<kFmt>((uint16_t)(hi >> 16));
  return pack2<kFmt>(a - fa, b - fb);
}

}  // namespace tc
}  // namespace mipnerf
