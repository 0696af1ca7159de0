// Shared device-side pieces of the persistent warpgroup-MMA network kernel (mlp_umma.cu: forward network / fused render
// kernel): shared-memory map, the barrier block, bounded waits, the weight ring and the split-bf16 store helpers.
#pragma once

#include "common.cuh"
#include "umma.cuh"

namespace dmnerf {
namespace uk {

using namespace umma;

constexpr int TILE_M = 128;                // rows per tile: two consumer warpgroups of 64 rows
constexpr int NS = 3;                      // weight ring stages
constexpr int STAGE_BYTES = 16384;         // up to [128 rows][64 bf16]
constexpr int CHUNK_BYTES = 16384;         // activation slab [128 rows][64 bf16]
constexpr int N_STEPS = 19;                 // 16 trunk half-steps, instance hidden, colour hidden (+ head on CUDA cores), instance head
constexpr int T_INS_HID = 16, T_RGB_HID = 17, T_INS_OUT = 18;
// fp32 side table of a network (KArgs::bias): per-step bias rows, then the small layers evaluated on CUDA cores
constexpr int B_WD = N_STEPS * 128;        // density_linear weights [256]
constexpr int B_BD = B_WD + 256;           // density bias (+3 pad)
constexpr int B_WRGB = B_BD + 4;           // rgb_linear weights [3][128]
constexpr int B_BRGB = B_WRGB + 3 * 128;   // rgb_linear bias (+1 pad)
constexpr int B_TOTAL = B_BRGB + 4;
constexpr int CONSUMERS = 256;             // two warpgroups: MMA issue, epilogues, prologue
constexpr int N_THREADS = CONSUMERS + 128; // + the producer warpgroup (its first warp streams the weights)
// Registers per thread after the role split (setmaxnreg): 128 x 24 + 256 x 240 = 64 512, the 168 x 384 of the launch
constexpr int PRODUCER_REGS = 24, CONSUMER_REGS = 240;
static_assert(128 * PRODUCER_REGS + CONSUMERS * CONSUMER_REGS <= 168 * N_THREADS, "register budget exceeds the launch's");
// Status code of the fp16 network in the error word (KArgs::status; the protocol errors are below 1000): an activation or an
// input exceeded the fp16 range
constexpr int STATUS_F16_RANGE = 1001;

// shared-memory map (offsets from the 1024-aligned base)
//   activation: 4 K chunks of the current 256-wide activation, each as a bf16 hi and a bf16 lo slab [128 rows][64]
//   (warpgroup g reads and writes rows [64 g, 64 g + 64)).  After the instance head the region holds the instance logits
//   of the tile (fused render kernel).
constexpr uint32_t SM_ACT = 0;
constexpr uint32_t ACT_CHUNK = 2 * CHUNK_BYTES;                  // hi slab, then lo slab
constexpr uint32_t SM_E_HI = SM_ACT + 4 * ACT_CHUNK;             // position embedding; the direction embedding after layer 5
constexpr uint32_t SM_E_LO = SM_E_HI + CHUNK_BYTES;
constexpr uint32_t SM_RING = SM_E_LO + CHUNK_BYTES;
constexpr uint32_t SM_MISC = SM_RING + NS * STAGE_BYTES;
constexpr uint32_t SM_FUSED = SM_MISC + 3072;                   // per-unit state of the fused render kernel
constexpr uint32_t SMEM_BYTES = SM_FUSED + 12288;
static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB shared memory of an SM");

struct Misc {                  // lives at SM_MISC
  uint64_t full[NS], empty[NS];
  int32_t abort_flag;
  float4 rowv[TILE_M];         // fused render kernel: per row rgb (xyz) and density (w) of the current tile
};
static_assert(sizeof(Misc) <= 3072, "Misc does not fit its shared-memory block");

// ------------------------------------------------------------------------------------------------ bounded waits
// Slow path of a barrier wait.  Inline, although it is cold: with a call in the consumer body, whose accumulators are live
// across it, ptxas fails register allocation at the CONSUMER_REGS budget (C7600).
// On a timeout the abort flag is raised and execution simply continues: every later wait returns at once, the kernel
// drains (with garbage results) and the host sees the status word -- no divergent early exits in the role loops.
__device__ __forceinline__ void slow_wait(uint64_t* bar, uint32_t parity, Misc* misc, int code, int32_t* status) {
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (*(volatile int32_t*)&misc->abort_flag) return;
    if (clock64() - t0 > 4000000000LL) {           // ~2 s: protocol failure
      atomicExch(&misc->abort_flag, code);
      atomicCAS(status, 0, code);
      return;
    }
  }
}
__device__ __forceinline__ void wait_bar(uint64_t* bar, uint32_t parity, Misc* misc, int code, int32_t* status) {
  if (!mbar_try_wait(bar, parity)) slow_wait(bar, parity, misc, code, status);
}

// Named barriers are executed by whole warps and are .aligned: reconverge first (the lanes of a warp can be in different
// convergence groups after a spin-wait; a warp arriving in two pieces would be counted twice).
template <int ID, int COUNT>
__device__ __forceinline__ void named_bar_sync() {
  __syncwarp();
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(COUNT) : "memory");
}
__device__ __forceinline__ void named_bar_sync_id(int id, int count) {
  __syncwarp();
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Position in the weight ring (warp-uniform).
struct Ring {
  uint32_t slot, phase;
  __device__ __forceinline__ void advance() {
    if (++slot == NS) { slot = 0; phase ^= 1; }
  }
};

// 8 fp32 values -> bf16 hi and bf16 lo into two K-major SW128 slabs (row `row`, K columns [k0, k0+8): one 16-byte unit each).
__device__ __forceinline__ void store_split8_smem(const float* vals, uint8_t* slab_hi, uint8_t* slab_lo, int row, int k0) {
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) split_bf16x2(vals[2 * j], vals[2 * j + 1], hi[j], lo[j]);
  const uint32_t o = sw128_offset(row, k0);
  *reinterpret_cast<uint4*>(slab_hi + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(slab_lo + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// fp16 network: 8 fp32 values -> fp16 into one K-major SW128 slab; returns the largest magnitude stored (range check).
__device__ __forceinline__ float store_f16x8_smem(const float* vals, uint8_t* slab, int row, int k0) {
  uint32_t h[4];
  float amax = 0.0f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    h[j] = pack_f16x2(vals[2 * j], vals[2 * j + 1]);
    amax = fmaxf(amax, fmaxf(fabsf(vals[2 * j]), fabsf(vals[2 * j + 1])));
  }
  *reinterpret_cast<uint4*>(slab + sw128_offset(row, k0)) = make_uint4(h[0], h[1], h[2], h[3]);
  return amax;
}

}  // namespace uk
}  // namespace dmnerf
