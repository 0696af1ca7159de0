// Thin inline-PTX layer over the Hopper tensor-core path (sm_90a): warpgroup MMA (wgmma.mma_async) with both operands in
// shared memory and the fp32 accumulator in registers, mbarrier, bulk async copy (TMA engine, 1-D).
// Layout conventions used everywhere in this library:
//   * K-major bf16 operand "slab": [rows][64 bf16] = 128 B per row, rows grouped by 8 into 1024 B swizzle atoms,
//     16-byte unit u of row r stored at unit (u ^ (r & 7))  (the canonical SWIZZLE_128B K-major layout).
//     A slab of R rows occupies R * 128 bytes and must start 1024 B aligned.
//   * wgmma shared-memory descriptor for such a slab: start address, LBO = 16 B (ignored for swizzled K-major),
//     SBO = 1024 B (stride between 8-row groups), layout type SWIZZLE_128B.  Advancing K by 16 elements inside the slab =
//     +32 B on the start address.  The same bytes read MN-major (rows = contraction index) take LBO = stride between
//     64-element MN blocks, SBO = 1024 B, and a K = 16 step advances the start address by 2048 B.
//   * accumulator fragment of m64nNk16 (fp32): thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and
//     columns 8 j + 2 (t % 4) (+ 1): d[4 j + 0, 1] = row r, columns c, c + 1; d[4 j + 2, 3] = row r + 8, same columns.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One lane of a converged warp (all 32 lanes must execute this).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor (SWIZZLE_128B) with explicit leading / stride byte offsets.
__device__ __forceinline__ uint64_t sdesc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);        // start address   bits [0,14)
  d |= (uint64_t)((lbo & 0x3FFFFu) >> 4) << 16;    // leading byte offset
  d |= (uint64_t)((sbo & 0x3FFFFu) >> 4) << 32;    // stride byte offset
  d |= (uint64_t)1 << 62;                          // layout type: SWIZZLE_128B
  return d;
}
// K-major SWIZZLE_128B slab starting at shared address `saddr`.
__device__ __forceinline__ uint64_t make_sdesc_sw128(uint32_t saddr) { return sdesc(saddr, 16, 1024); }

// Byte offset of element (row, k) inside a K-major SW128 slab (k in [0,64)).
__host__ __device__ __forceinline__ uint32_t sw128_offset(int row, int k) {
  const int unit = (k >> 3) ^ (row & 7);
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + unit * 16 + (k & 7) * 2);
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: returns false (and the caller must bail out) instead of hanging the GPU if the barrier never flips.
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, uint32_t max_spins = 1u << 26) {
  for (uint32_t i = 0; i < max_spins; ++i)
    if (mbar_try_wait(bar, parity)) return true;
  return false;
}

// ---------------------------------------------------------------- proxies / fences
// Generic-proxy shared-memory writes (operand slabs stored by threads) made visible to the tensor core (async proxy).
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- bulk async copy (TMA engine, 1-D)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------- warpgroup MMA (all 128 threads of a warpgroup)
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Keeps the compiler from moving accumulator reads / writes across an asynchronous MMA.
template <int R>
__device__ __forceinline__ void wg_reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T; TA / TB = 1: that operand is MN-major.  scale_d = 0 overwrites D.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,"
      "%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31},"
      " %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

// ---------------------------------------------------------------- bf16 hi/lo split (round-to-nearest)
// x ~= hi + lo with hi = bf16(x), lo = bf16(x - hi): 16 significand bits in total.
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// Two values -> packed (hi0,hi1) and (lo0,lo1) words (element 0 in the low half-word).
__device__ __forceinline__ void split_bf16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  const float2 hf = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

}  // namespace umma
