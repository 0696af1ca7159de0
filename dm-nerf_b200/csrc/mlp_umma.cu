// Warpgroup-MMA (wgmma) implementation of the DM_NeRF network for one 128-sample tile per CTA (persistent, 1 CTA / SM).
//
// Arithmetic: every fp32 operand is split into bf16 hi + bf16 lo (16 significand bits); each algorithmic GEMM is issued
// as three tensor passes  A_hi*W_hi + A_lo*W_hi + A_hi*W_lo  accumulating in fp32 registers (relative error ~2^-16 per
// product, ~1e-5 on outputs, inside the 1e-4 parity budget; single-pass bf16/tf32 is not).
//
// Data flow per tile (nothing 256-wide ever leaves the SM):
//   * activations: the current 256-wide activation lives in shared memory as split bf16 (4 K chunks x hi / lo slabs in the
//     128-byte-swizzled K-major layout the tensor core reads).  Each of the two consumer warpgroups owns 64 rows of the tile;
//     a 256-wide layer is two N = 128 half-steps accumulated into two register accumulators, and the epilogue (bias, ReLU,
//     split) overwrites the activation in place once the layer's MMAs have completed.
//   * the position embedding is a shared-memory slab of its own (layers 0 and 5); after layer 5 the direction embedding
//     replaces it (colour hidden layer).
//   * weights: packed once per weight update (dmnerf_set_weights) into the exact shared-memory image, streamed in 16 KB
//     stages through a ring with 1-D bulk async copies (TMA engine, mbarrier completion) from L2 by one producer warp; both
//     warpgroups read every stage, and a stage is handed back when the MMAs of both have completed.
//   * heads: rgb_feature_linear / ins_feature_linear have no activation, so they are folded into the following layer at
//     pack time (W' = W2 W1, fp64 accumulate); density (N=1) and the 3-wide rgb head are fp32 CUDA-core dot products in the
//     epilogues of layer 7 / the colour hidden layer; the instance head is one more MMA.  19 half-steps per tile.
// All waits are bounded: a protocol bug raises an error code, never a hang.
//
#include <cstring>
#include <type_traits>
#include <vector>

#include "ray_ops.cuh"
#include "uk_pipe.cuh"
#include "umma_api.cuh"

namespace dmnerf {
namespace uk {

using namespace umma;
enum ChunkKind : int8_t { CK_E = 6, CK_D = 7 };              // 0..3 = activation K chunk

struct Step {
  int8_t n_chunks;
  int8_t chunk[MAX_CHUNKS];   // ChunkKind or activation chunk
  int8_t dep[MAX_CHUNKS];     // tile-relative step whose epilogue produces the chunk; -1 = tile inputs
  int8_t ksteps[MAX_CHUNKS];  // K/16 MMAs for this chunk (4, or 2 for the direction embedding)
  int8_t out_slot;            // destination half of the activation, or -1 = network outputs
  int8_t relu;
  int16_t n;                  // rows of the packed weight stage (multiple of 16, <= 128)
};

struct Program {
  Step step[N_STEPS];
  uint32_t stage_off[MAX_STAGES];     // byte offset of every weight stage in the packed image
  int32_t n_stages;
  int32_t ins_num;
};

// Shared state of the fused render kernel: one work unit = 2 rays = 1 coarse tile (2 x 64 samples) + 3 fine tiles (2 x 192).
constexpr int FS = 64, FI = 128, FF = FS + FI;        // the fused path is specialised for 64 + 128 samples
constexpr int ACC_W = 5 + DMNERF_MAX_INS + 1 + 3;      // rgb3, depth, acc, ins_num+1 (padded)
struct Fused {
  float ray[2][8];            // per ray: o(3), d(3), |d|, valid
  float zc[2][FS];            // coarse depths (after jitter)
  float zf[2][FF];            // fine depths (sorted union)
  float w[TILE_M];            // compositing weights of the current tile's rows
  float tot[4];               // per-warp transmittance products of the current tile
  float carry[4][2];          // transmittance entering fine tile j (rays A, B)
  float accum[2][6][ACC_W];   // per ray and 32-sample chunk: partial sums of rgb3, depth, acc, instance logits (each slot has
                              // exactly one writer and the chunks are added in order: bit-reproducible, no atomics)
  float bins[2][FS], cdf[2][FS], vals[2][FF];
};
static_assert(sizeof(Fused) <= 12288, "Fused state does not fit its shared-memory block");

struct KArgs {
  const uint8_t* image;        // packed bf16 operand image (fused: coarse network)
  const float* bias;           // [N_STEPS][128] step biases, then the B_* blocks above
  const uint8_t* image_fine;   // fused: fine network
  const float* bias_fine;
  // fused render inputs / outputs (any output may be NULL)
  const float* z_in; int64_t z_stride; const float* t_rand; const float* u;
  int64_t n_rays; int32_t keep_all_ins;
  float* rgb_c; float* rgb_f; float* depth_c; float* depth_f; float* acc_c; float* acc_f; float* ins_c; float* ins_f;
  float* zc_out; float* zf_out; float* wc_out; float* wf_out;
  const float* x;              // [M, 90] or nullptr
  const float* rays_o; const float* rays_d; const float* z;   // rays mode
  int64_t m;
  int32_t s;                   // samples per ray (rays mode)
  float* out;                  // [M, C]
  float* acts;                 // training forward (RAW mode): ActPlanes base, or nullptr
  int32_t* status;             // device error word
};

// ------------------------------------------------------------------------------------------------ prologue helpers
// sin and cos of one argument with |a| < ~1e5: three-constant Cody-Waite reduction by pi/2 + the single-precision minimax
// polynomials on [-pi/4, pi/4] (the textbook algorithm behind the library's own fast path, <= 2 ulp), written without the
// large-argument branch so that the compiler can interleave the independent evaluations of a row.
__device__ __forceinline__ void sincos_cw(float a, float& sn, float& cs) {
  const float t = fmaf(a, 0.636619772f, 12582912.0f);          // 1.5 * 2^23: the integer n = rint(a * 2/pi) lands in the mantissa
  const int n = __float_as_int(t);
  const float j = t - 12582912.0f;
  float r = fmaf(j, -1.57079601e+00f, a);
  r = fmaf(j, -3.13916473e-07f, r);
  r = fmaf(j, -5.39030253e-15f, r);
  const float r2 = r * r;
  float ps = fmaf(-1.9515295891e-4f, r2, 8.3321608736e-3f);
  ps = fmaf(ps, r2, -1.6666654611e-1f);
  const float sr = fmaf(r * r2, ps, r);
  float pc = fmaf(2.443315711809948e-5f, r2, -1.388731625493765e-3f);
  pc = fmaf(pc, r2, 4.166664568298827e-2f);
  pc = fmaf(pc, r2, -0.5f);
  const float cr = fmaf(r2, pc, 1.0f);
  float s0 = (n & 1) ? cr : sr, c0 = (n & 1) ? sr : cr;
  sn = (n & 2) ? -s0 : s0;
  cs = ((n + 1) & 2) ? -c0 : c0;
}

// Elements [E0, E0 + COUNT) of the embedding [v, sin(2^0 v), cos(2^0 v), ..., sin(2^(L-1) v), cos(2^(L-1) v)].
// FAST: every argument is known to be small enough for sincos_cw (checked warp-wide by the caller).
template <int E0, int COUNT, int L, bool FAST>
__device__ __forceinline__ void fill_embedding(const float v[3], float* vals /* COUNT */) {
  constexpr int F_LO = (E0 <= 3) ? 0 : (E0 - 3) / 6;
  constexpr int F_HI_RAW = (E0 + COUNT - 1 - 3) / 6;
  constexpr int F_HI = (E0 + COUNT - 1 < 3) ? -1 : (F_HI_RAW < L - 1 ? F_HI_RAW : L - 1);
#pragma unroll
  for (int i = 0; i < COUNT; ++i) vals[i] = 0.0f;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    if (c >= E0 && c < E0 + COUNT) vals[c - E0] = v[c];
#pragma unroll
  for (int f = F_LO; f <= F_HI; ++f) {
    const float sc = (float)(1 << f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int es = 3 + 6 * f + c, ec = es + 3;
      const bool use_s = es >= E0 && es < E0 + COUNT, use_c = ec >= E0 && ec < E0 + COUNT;
      if (use_s || use_c) {
        float sn, cs;
        if (FAST) sincos_cw(v[c] * sc, sn, cs);
        else sincosf(v[c] * sc, &sn, &cs);
        if (use_s) vals[es - E0] = sn;
        if (use_c) vals[ec - E0] = cs;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ the kernel
// Warps 0-7: two consumer warpgroups (MMA issue, epilogues, prologue); warp 8: weight producer.
template <bool FUSED>
__global__ void __launch_bounds__(N_THREADS, 1) mlp_umma_kernel(const __grid_constant__ Program prog, const KArgs a) {
  // The kernel has no static shared memory, so the dynamic block starts at offset 0 of the CTA's shared window and
  // is 1024-aligned by construction (checked below).
  extern __shared__ __align__(1024) uint8_t smem[];
  Misc* misc = reinterpret_cast<Misc*>(smem + SM_MISC);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // RAW: work item = one 128-row tile of a.m samples.  FUSED: work item = ray pair = 4 tiles (1 coarse + 3 fine).
  const int64_t n_items = FUSED ? (a.n_rays + 1) / 2 : (a.m + TILE_M - 1) / TILE_M;
  const int64_t my_items = (n_items > blockIdx.x) ? (n_items - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const int64_t my_tiles = FUSED ? 4 * my_items : my_items;
  Fused* fz = reinterpret_cast<Fused*>(smem + SM_FUSED);
  const int C = 4 + prog.ins_num + 1;

  if (tid == 0) {
    for (int i = 0; i < NS; ++i) { mbar_init(&misc->full[i], 1); mbar_init(&misc->empty[i], 8); }
    misc->abort_flag = 0;
    fence_barrier_init();
  }
  __syncthreads();
  if ((smem_u32(smem) & 1023u) != 0) {
    if (tid == 0) { atomicExch(&misc->abort_flag, 901); atomicCAS(a.status, 0, 901); }
  }

  if (warp == 8) {
    // =========================================================== weight producer (converged warp, one elected lane issues)
    Ring ring{0, 0};
    const int n_stages = prog.n_stages;
    for (int64_t ti = 0; ti < my_tiles; ++ti) {
      const uint8_t* image = (FUSED && (ti & 3) != 0) ? a.image_fine : a.image;
      for (int si = 0; si < n_stages; ++si) {
        const uint32_t off = prog.stage_off[si], bytes = prog.stage_off[si + 1] - off;
        wait_bar(&misc->empty[ring.slot], ring.phase ^ 1, misc, 101, a.status);
        if (elect_one()) {
          mbar_arrive_expect_tx(&misc->full[ring.slot], bytes);
          bulk_g2s(smem + SM_RING + ring.slot * STAGE_BYTES, image + off, bytes, &misc->full[ring.slot]);
        }
        __syncwarp();
        ring.advance();
      }
    }
    return;
  }

  // =========================================================== consumer warpgroups
  const int g = tid >> 7;                       // warpgroup: tile rows [64 g, 64 g + 64)
  const int wl = warp & 3;
  const int ra = 64 * g + 16 * wl + (lane >> 2);  // tile rows of this thread's accumulator fragment: ra, ra + 8
  const int q4 = lane & 3;                      // fragment columns 8 j + 2 q4 (+ 1)
  const int pr = 64 * g + (tid & 63);           // prologue: tile row of this thread
  const int ph = (tid >> 6) & 1;                // prologue: which half of the row's embedding columns
  const int bar_wg = 1 + g;                     // named barrier of this warpgroup
  uint8_t *e_hi = smem + SM_E_HI, *e_lo = smem + SM_E_LO;
  const uint32_t ring_base = smem_u32(smem + SM_RING);
  const uint32_t act_base = smem_u32(smem + SM_ACT) + 8192u * g;     // this warpgroup's 64 rows inside every slab
  const uint32_t e_base = smem_u32(e_hi) + 8192u * g;
  Ring ring{0, 0};
  int prev_slot = -1;
  float acc0[64], acc1[64];

  // One weight stage: wait for it, issue its MMAs (A_hi * W and, for a W_hi stage, A_lo * W), hand the previous stage back
  // once its MMAs have completed (the ring holds the stage in flight, the stage issued before it and the one being filled).
  auto stage = [&](float (&acc)[64], uint32_t a_hi, uint32_t a_lo, bool with_lo, int ks, uint32_t scale0) {
    const uint32_t s = ring.slot;
    wait_bar(&misc->full[s], ring.phase, misc, 204, a.status);
    const uint32_t w = ring_base + s * STAGE_BYTES;
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k < ks) {
        wgmma_n128<0, 0>(acc, make_sdesc_sw128(a_hi + 32 * k), make_sdesc_sw128(w + 32 * k), k == 0 ? scale0 : 1u);
        if (with_lo) wgmma_n128<0, 0>(acc, make_sdesc_sw128(a_lo + 32 * k), make_sdesc_sw128(w + 32 * k), 1u);
      }
    }
    wg_commit();
    wg_wait<1>();
    if (prev_slot >= 0 && lane == 0) mbar_arrive(&misc->empty[prev_slot]);
    prev_slot = (int)s;
    ring.advance();
  };
  auto drain = [&]() {
    wg_wait<0>();
    wg_reg_fence(acc0);
    wg_reg_fence(acc1);
    if (prev_slot >= 0 && lane == 0) mbar_arrive(&misc->empty[prev_slot]);
    prev_slot = -1;
  };
  // One 64-wide K chunk (W_hi stage, then W_lo stage) of a half-step
  auto chunk = [&](float (&acc)[64], uint32_t a_hi, uint32_t a_lo, int ks, bool first) {
    stage(acc, a_hi, a_lo, true, ks, first ? 0u : 1u);
    stage(acc, a_hi, a_lo, false, ks, 1u);
  };
  auto act_chunk = [&](float (&acc)[64], int c, bool first) {
    const uint32_t hi = act_base + c * ACT_CHUNK;
    chunk(acc, hi, hi + CHUNK_BYTES, 4, first);
  };
  auto all_act = [&](float (&acc)[64]) { for (int c = 0; c < 4; ++c) act_chunk(acc, c, c == 0); };
  auto e_chunk = [&](float (&acc)[64], int ks, bool first) { chunk(acc, e_base, e_base + CHUNK_BYTES, ks, first); };
  auto wg_sync = [&]() { named_bar_sync_id(bar_wg, 128); };
  auto all_sync = [&]() { named_bar_sync<3, CONSUMERS>(); };

  for (int64_t ti = 0; ti < my_tiles; ++ti) {
    const int j = FUSED ? (int)(ti & 3) : 0;                            // fused: 0 = coarse tile, 1..3 = fine tiles
    const int64_t item = blockIdx.x + (FUSED ? (ti >> 2) : ti) * gridDim.x;
    const float* bias_base = (FUSED && j != 0) ? a.bias_fine : a.bias;
    // ---------------- rows of this tile: which sample a tile row is
    auto row_of = [&](int r, int& rl, int& si, int64_t& row, bool& valid) {
      if constexpr (FUSED) {
        if (j == 0) { rl = r >> 6; si = r & 63; }
        else { const int gr = (j - 1) * TILE_M + r; rl = gr / FF; si = gr % FF; }
        row = 0;
        valid = fz->ray[rl][7] != 0.0f;
      } else {
        rl = 0; si = 0;
        row = item * TILE_M + r;
        valid = row < a.m;
      }
    };
    // ---------------- prologue: points + position embedding of row pr, columns [32 ph, 32 ph + 32)
    if (FUSED && j == 0) {
      if (tid < 2) {
        const int64_t ray = item * 2 + tid;
        const bool ok = ray < a.n_rays;
        float* rs = fz->ray[tid];
        for (int c = 0; c < 3; ++c) { rs[c] = ok ? a.rays_o[ray * 3 + c] : 0.0f; rs[3 + c] = ok ? a.rays_d[ray * 3 + c] : 0.0f; }
        rs[6] = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(rs[3], rs[3]), __fmul_rn(rs[4], rs[4])), __fmul_rn(rs[5], rs[5])));
        rs[7] = ok ? 1.0f : 0.0f;
      }
      all_sync();
    }
    int p_rl, p_si;
    int64_t p_row;
    bool p_valid;
    row_of(pr, p_rl, p_si, p_row, p_valid);
    float pt[3] = {0.f, 0.f, 0.f}, vd[3] = {0.f, 0.f, 0.f};
    auto save_emb = [&](int col0, const float* vals, int cnt) {          // training forward: keep the embedded inputs
      if constexpr (!FUSED) {
        if (a.acts && p_valid) {
          float* dst = act_planes(a.acts, a.m).emb + (int64_t)col0 * a.m + p_row;      // column-major [90][M]
          for (int i = 0; i < cnt; ++i)
            if (col0 + i < CH_IN && (col0 >= CH_POS || col0 + i < CH_POS)) dst[(int64_t)i * a.m] = vals[i];
        }
      }
    };
    {
      float vals[32];
      if (!FUSED && a.x) {
#pragma unroll
        for (int i = 0; i < 32; ++i) vals[i] = (p_valid && 32 * ph + i < CH_POS) ? a.x[p_row * CH_IN + 32 * ph + i] : 0.0f;
      } else {
        if (p_valid) {
          float o0, o1, o2, d0, d1, d2, nrm, zz;
          if constexpr (FUSED) {
            const float* rs = fz->ray[p_rl];
            o0 = rs[0]; o1 = rs[1]; o2 = rs[2]; d0 = rs[3]; d1 = rs[4]; d2 = rs[5]; nrm = rs[6];
            if (j == 0) {
              // render.py:40-47: shared / per-ray coarse row, jittered inside its stratum when t_rand is given
              const int64_t ray = item * 2 + p_rl;
              const float* zr = a.z_in + ray * a.z_stride;
              zz = zr[p_si];
              if (a.t_rand) {
                const float lower = (p_si == 0) ? zz : __fmul_rn(0.5f, __fadd_rn(zz, zr[p_si - 1]));
                const float upper = (p_si == FS - 1) ? zz : __fmul_rn(0.5f, __fadd_rn(zr[p_si + 1], zz));
                zz = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), a.t_rand[ray * FS + p_si]));
              }
              if (ph == 0) {
                fz->zc[p_rl][p_si] = zz;
                if (a.zc_out) a.zc_out[ray * FS + p_si] = zz;
              }
            } else {
              zz = fz->zf[p_rl][p_si];
            }
          } else {
            // rays mode: sample s of ray r at depth z.  Points mode (z == NULL, s == 1): rays_o holds the query points and
            // rays_d the view directions exactly as they go into the embedding (mesh_generator.py:40-44 passes zeros).
            const int64_t ray = p_row / a.s;
            zz = a.z ? a.z[p_row] : 0.0f;
            o0 = a.rays_o[ray * 3]; o1 = a.rays_o[ray * 3 + 1]; o2 = a.rays_o[ray * 3 + 2];
            d0 = a.rays_d[ray * 3]; d1 = a.rays_d[ray * 3 + 1]; d2 = a.rays_d[ray * 3 + 2];
            nrm = a.z ? sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2))) : 1.0f;
          }
          if (FUSED || a.z) {
            pt[0] = __fadd_rn(o0, __fmul_rn(d0, zz));      // render.py:49
            pt[1] = __fadd_rn(o1, __fmul_rn(d1, zz));
            pt[2] = __fadd_rn(o2, __fmul_rn(d2, zz));
          } else {
            pt[0] = o0; pt[1] = o1; pt[2] = o2;
          }
          vd[0] = __fdiv_rn(d0, nrm); vd[1] = __fdiv_rn(d1, nrm); vd[2] = __fdiv_rn(d2, nrm);      // render.py:37
        }
        // |2^9 x| small enough for the branch-free sin/cos in every lane?  (warp-uniform choice; scenes are a few units wide)
        const float amax = fmaxf(fmaxf(fabsf(pt[0]), fabsf(pt[1])), fabsf(pt[2]));
        const bool fast = __all_sync(0xffffffffu, amax < 64.0f);
        if (ph == 0) { if (fast) fill_embedding<0, 32, L_POS, true>(pt, vals); else fill_embedding<0, 32, L_POS, false>(pt, vals); }
        else { if (fast) fill_embedding<32, 32, L_POS, true>(pt, vals); else fill_embedding<32, 32, L_POS, false>(pt, vals); }
        if (!p_valid) {
#pragma unroll
          for (int i = 0; i < 32; ++i) vals[i] = 0.0f;
        }
      }
      save_emb(32 * ph, vals, 32);
#pragma unroll
      for (int u = 0; u < 4; ++u) store_split8_smem(vals + 8 * u, e_hi, e_lo, pr, 32 * ph + 8 * u);
    }
    fence_proxy_async_smem();            // the embeddings are read by the tensor core through the async proxy
    wg_sync();

    // ---------------- epilogue helpers
    const float* bias_t = bias_base;
    const ActPlanes ap = act_planes(a.acts, a.m);
    int64_t row_ab[2];
    bool valid_ab[2];
    {
      int rl_, si_;
      row_of(ra, rl_, si_, row_ab[0], valid_ab[0]);
      row_of(ra + 8, rl_, si_, row_ab[1], valid_ab[1]);
    }
    // bias + ReLU of one 128-column half-step accumulator; store as split bf16 into activation half `half` (or nowhere)
    auto hidden = [&](float (&acc)[64], int t, int half, int plane, int width, int col_off) {
      const float* bias = bias_t + t * 128;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const int col = 8 * jj + 2 * q4;
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          acc[4 * jj + 2 * h] = fmaxf(acc[4 * jj + 2 * h] + bb.x, 0.0f);
          acc[4 * jj + 2 * h + 1] = fmaxf(acc[4 * jj + 2 * h + 1] + bb.y, 0.0f);
          if (half >= 0) {
            uint32_t hi, lo;
            split_bf16x2(acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1], hi, lo);
            const int c256 = 128 * half + col;
            const uint32_t o = SM_ACT + (c256 >> 6) * ACT_CHUNK + sw128_offset(ra + 8 * h, c256 & 63);
            *reinterpret_cast<uint32_t*>(smem + o) = hi;
            *reinterpret_cast<uint32_t*>(smem + o + CHUNK_BYTES) = lo;
          }
        }
      }
      if constexpr (!FUSED) {
        if (a.acts) {                            // training forward: keep the post-activation values and their ReLU masks
          float* base = (plane < 8) ? ap.h[plane] : (plane == 8 ? ap.rgb_hid : ap.ins_hid);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!valid_ab[h]) continue;
            float* dst = base + row_ab[h] * width + col_off + 2 * q4;
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
              *reinterpret_cast<float2*>(dst + 8 * jj) = make_float2(acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1]);
          }
#pragma unroll
          for (int grp = 0; grp < 8; ++grp) {      // 16 units = n8 blocks 2 grp, 2 grp + 1
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              uint32_t b = 0;
              b |= (acc[4 * (2 * grp) + 2 * h] > 0.0f ? 1u : 0u) << (2 * q4);
              b |= (acc[4 * (2 * grp) + 2 * h + 1] > 0.0f ? 1u : 0u) << (2 * q4 + 1);
              b |= (acc[4 * (2 * grp + 1) + 2 * h] > 0.0f ? 1u : 0u) << (8 + 2 * q4);
              b |= (acc[4 * (2 * grp + 1) + 2 * h + 1] > 0.0f ? 1u : 0u) << (9 + 2 * q4);
              b |= __shfl_xor_sync(0xffffffffu, b, 1);
              b |= __shfl_xor_sync(0xffffffffu, b, 2);
              if (q4 == 0 && valid_ab[h]) ap.bits[act_bits_index(plane, (col_off >> 4) + grp, row_ab[h], a.m)] = (uint16_t)b;
            }
          }
        }
      }
    };
    // sum over the four lanes of a quad (the four column owners of a row), fixed order
    auto quad_sum = [&](float v) { v += __shfl_xor_sync(0xffffffffu, v, 1); v += __shfl_xor_sync(0xffffffffu, v, 2); return v; };

    // ---------------- trunk: layers 0..7
    float dens[2] = {0.f, 0.f};
    for (int l = 0; l < 8; ++l) {
      if (l == 0) { e_chunk(acc0, 4, true); e_chunk(acc1, 4, true); }
      else {
        all_act(acc0); if (l == 5) e_chunk(acc0, 4, false);
        all_act(acc1); if (l == 5) e_chunk(acc1, 4, false);
      }
      drain();
      wg_sync();                                   // every warp's MMAs on the old activation have completed
      hidden(acc0, 2 * l, 0, l, W_HID, 0);
      hidden(acc1, 2 * l + 1, 1, l, W_HID, 128);
      if (l == 7) {                                // density_linear (dm_nerf.py:101) on the final trunk activation
        const float* wd = bias_t + B_WD;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int col = 8 * jj + 2 * q4;
          const float2 w0 = __ldg(reinterpret_cast<const float2*>(wd + col)), w1 = __ldg(reinterpret_cast<const float2*>(wd + 128 + col));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            dens[h] = fmaf(acc0[4 * jj + 2 * h], w0.x, dens[h]); dens[h] = fmaf(acc0[4 * jj + 2 * h + 1], w0.y, dens[h]);
            dens[h] = fmaf(acc1[4 * jj + 2 * h], w1.x, dens[h]); dens[h] = fmaf(acc1[4 * jj + 2 * h + 1], w1.y, dens[h]);
          }
        }
      }
      if (l == 5) {
        // the position embedding has been read for the last time: the direction embedding takes its place (columns 0..31)
        float vals[16];
        if (!FUSED && a.x) {
#pragma unroll
          for (int i = 0; i < 16; ++i) vals[i] = (p_valid && 16 * ph + i < CH_DIR) ? a.x[p_row * CH_IN + CH_POS + 16 * ph + i] : 0.0f;
        } else {
          if (ph == 0) fill_embedding<0, 16, L_DIR, true>(vd, vals); else fill_embedding<16, 16, L_DIR, true>(vd, vals);
          if (!p_valid) {
#pragma unroll
            for (int i = 0; i < 16; ++i) vals[i] = 0.0f;
          }
        }
        save_emb(CH_POS + 16 * ph, vals, 16);
        store_split8_smem(vals, e_hi, e_lo, pr, 16 * ph);
        store_split8_smem(vals + 8, e_hi, e_lo, pr, 16 * ph + 8);
      }
      fence_proxy_async_smem();
      wg_sync();
    }
    // ---------------- folded instance hidden layer (acc0) and folded colour hidden layer [h | dir] (acc1)
    all_act(acc0);
    all_act(acc1); e_chunk(acc1, 2, false);
    drain();
    wg_sync();
    float rgb[2][3];
    hidden(acc1, T_RGB_HID, -1, 8, W_HID / 2, 0);
    {
      // rgb_linear (dm_nerf.py:102,105) on CUDA cores
#pragma unroll
      for (int h = 0; h < 2; ++h) rgb[h][0] = rgb[h][1] = rgb[h][2] = 0.0f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const int col = 8 * jj + 2 * q4;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float2 w = __ldg(reinterpret_cast<const float2*>(bias_t + B_WRGB + c * 128 + col));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            rgb[h][c] = fmaf(acc1[4 * jj + 2 * h], w.x, rgb[h][c]);
            rgb[h][c] = fmaf(acc1[4 * jj + 2 * h + 1], w.y, rgb[h][c]);
          }
        }
      }
    }
    hidden(acc0, T_INS_HID, 0, 9, W_HID / 2, 0);
    fence_proxy_async_smem();
    wg_sync();
    // ---------------- instance head (dm_nerf.py:103,105) on the instance hidden activation (activation half 0)
    // The weight stages of this step hold n = pad16(ins_num + 1) rows, but the MMA is issued with N = 128 like every other
    // step: rows n..127 of the ring slot are stale bytes of an earlier stage.  Output column c depends only on B row c, so
    // columns >= n are garbage and are never read (only columns < ins_num + 1 are stored below).  The head is 1 of 19
    // half-steps of a tile.
    act_chunk(acc0, 0, true); act_chunk(acc0, 1, false);
    drain();
    wg_sync();
    const int n_ins1 = prog.ins_num + 1;
    float c3[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      c3[h][0] = quad_sum(rgb[h][0]) + __ldg(bias_t + B_BRGB + 0);
      c3[h][1] = quad_sum(rgb[h][1]) + __ldg(bias_t + B_BRGB + 1);
      c3[h][2] = quad_sum(rgb[h][2]) + __ldg(bias_t + B_BRGB + 2);
      c3[h][3] = quad_sum(dens[h]) + __ldg(bias_t + B_BD);
    }
    const float* bias_ins = bias_t + T_INS_OUT * 128;
    if constexpr (!FUSED) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!valid_ab[h]) continue;
        float* o = a.out + row_ab[h] * C;
        if (q4 == 0) { o[0] = c3[h][0]; o[1] = c3[h][1]; o[2] = c3[h][2]; o[3] = c3[h][3]; }
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int col = 8 * jj + 2 * q4;
          if (col < n_ins1) o[4 + col] = acc0[4 * jj + 2 * h] + __ldg(bias_ins + col);
          if (col + 1 < n_ins1) o[5 + col] = acc0[4 * jj + 2 * h + 1] + __ldg(bias_ins + col + 1);
        }
      }
    } else {
      // per-row outputs into shared memory: rgb / density in misc->rowv, instance logits [128][128] over the activation
      float* logit = reinterpret_cast<float*>(smem + SM_ACT);
      all_sync();                        // both warpgroups' instance-head MMAs have read the activation
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (q4 == 0) misc->rowv[ra + 8 * h] = make_float4(c3[h][0], c3[h][1], c3[h][2], c3[h][3]);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int col = 8 * jj + 2 * q4;
          if (col < n_ins1) logit[(ra + 8 * h) * 128 + col] = acc0[4 * jj + 2 * h] + __ldg(bias_ins + col);
          if (col + 1 < n_ins1) logit[(ra + 8 * h) * 128 + col + 1] = acc0[4 * jj + 2 * h + 1] + __ldg(bias_ins + col + 1);
        }
      }
      all_sync();
      if (tid < TILE_M) {
        // ---- sigma -> alpha -> transmittance (render.py:7-18): warp scan + cross-warp carry; thread = tile row
        const int r = tid;
        int rl, si;
        int64_t row_unused;
        bool valid;
        row_of(r, rl, si, row_unused, valid);
        const int S = (j == 0) ? FS : FF;
        const float4 rv = misc->rowv[r];
        const float* zs = (j == 0) ? fz->zc[rl] : fz->zf[rl];
        const float zi = zs[si];
        float dist = (si == S - 1) ? 1e10f : __fsub_rn(zs[si + 1], zi);
        dist = __fmul_rn(dist, fz->ray[rl][6]);
        const float alpha = __fsub_rn(1.0f, expf(-__fmul_rn(fmaxf(rv.w, 0.0f), dist)));
        const float f = __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f);
        const int lane_i = r & 31, wi = r >> 5;
        const float incl = warp_scan_mul(f, lane_i);
        float excl = __shfl_up_sync(FULL, incl, 1);
        if (lane_i == 0) excl = 1.0f;
        if (lane_i == 31) fz->tot[wi] = incl;
        named_bar_sync<4, 128>();
        // transmittance entering this warp = carry of the ray x products of earlier warps of the same ray in this tile
        const int first_w = (j == 0) ? (rl * 2) : ((j == 2) ? (rl * 2) : 0);   // first warp of my ray inside this tile
        float pre = (j >= 2) ? fz->carry[j][rl] : 1.0f;
        for (int w2 = first_w; w2 < wi; ++w2) pre = __fmul_rn(pre, fz->tot[w2]);
        const float wgt = valid ? __fmul_rn(alpha, __fmul_rn(pre, excl)) : 0.0f;
        fz->w[r] = wgt;
        if (j >= 1 && j <= 2 && wi == 0 && lane_i < 2) {
          // carry into the next fine tile for ray `lane_i` (ray A ends inside tile 2, ray B starts there)
          float cpre = (j == 2) ? fz->carry[2][lane_i] : 1.0f;
          const int wa = (j == 1) ? (lane_i == 0 ? 0 : 4) : (lane_i == 0 ? 0 : 2);    // warps of that ray in this tile
          const int wb = (j == 1) ? (lane_i == 0 ? 4 : 4) : (lane_i == 0 ? 2 : 4);
          for (int w2 = wa; w2 < wb; ++w2) cpre = __fmul_rn(cpre, fz->tot[w2]);
          fz->carry[j + 1][lane_i] = cpre;
        }
        if (j == 0 && a.wc_out && valid) a.wc_out[(item * 2 + rl) * FS + si] = wgt;
        if (j != 0 && a.wf_out && valid) a.wf_out[(item * 2 + rl) * FF + si] = wgt;
        // ---- weighted sums (render.py:19-20 + acc): warp reduce per 32-sample chunk
        float p0 = __fmul_rn(wgt, sigmoidf_acc(rv.x)), p1 = __fmul_rn(wgt, sigmoidf_acc(rv.y)), p2 = __fmul_rn(wgt, sigmoidf_acc(rv.z));
        float p3 = __fmul_rn(wgt, zi), p4 = wgt;
        p0 = warp_sum(p0); p1 = warp_sum(p1); p2 = warp_sum(p2); p3 = warp_sum(p3); p4 = warp_sum(p4);
        float* ac = fz->accum[rl][si >> 5];
        if (lane_i == 0) { ac[0] = p0; ac[1] = p1; ac[2] = p2; ac[3] = p3; ac[4] = p4; }
        named_bar_sync<4, 128>();        // weights of the tile complete
        // instance logits weighted by the (detached) weights: sum_i w_i raw_i[4+k] (render.py:22-24); lane = channel,
        // the 32 rows of this warp's chunk added in order
        for (int ch = lane_i; ch < n_ins1; ch += 32) {
          float sacc = 0.0f;
          for (int rr = 0; rr < 32; ++rr) sacc = __fadd_rn(sacc, __fmul_rn(fz->w[32 * wi + rr], logit[(32 * wi + rr) * 128 + ch]));
          ac[5 + ch] = sacc;
        }
        named_bar_sync<4, 128>();        // all running sums of this tile are in
        // ---- rays that end in this tile: write their maps (render.py:19-26) and clear the sums
        const int done_lo = (j == 0) ? 0 : ((j == 2) ? 0 : ((j == 3) ? 1 : 2));
        const int done_hi = (j == 0) ? 2 : ((j == 2) ? 1 : ((j == 3) ? 2 : 2));
        for (int rr = done_lo; rr < done_hi; ++rr) {
          const int64_t ray = item * 2 + rr;
          if (fz->ray[rr][7] == 0.0f) continue;
          for (int e = r; e < 5 + n_ins1; e += TILE_M) {
            float vsum = 0.0f;
            for (int cj = 0; cj < S / 32; ++cj) vsum = __fadd_rn(vsum, fz->accum[rr][cj][e]);
            float* o_rgb = (j == 0) ? a.rgb_c : a.rgb_f;
            float* o_dep = (j == 0) ? a.depth_c : a.depth_f;
            float* o_acc = (j == 0) ? a.acc_c : a.acc_f;
            float* o_ins = (j == 0) ? a.ins_c : a.ins_f;
            const int n_out = a.keep_all_ins ? n_ins1 : n_ins1 - 1;
            if (e < 3) { if (o_rgb) o_rgb[ray * 3 + e] = vsum; }
            else if (e == 3) { if (o_dep) o_dep[ray] = vsum; }
            else if (e == 4) { if (o_acc) o_acc[ray] = vsum; }
            else if (e - 5 < n_out) { if (o_ins) o_ins[ray * n_out + (e - 5)] = sigmoidf_acc(vsum); }
          }
        }
        if (j == 0) {
          // ---- hierarchical sampling (render.py:66-70): 64 threads per ray, results stay in shared memory
          const int rr = r >> 6, t64 = r & 63;
          fz->vals[rr][t64] = fz->zc[rr][t64];
          if (t64 < FS - 1) fz->bins[rr][t64] = __fmul_rn(0.5f, __fadd_rn(fz->zc[rr][t64 + 1], fz->zc[rr][t64]));
          named_bar_sync<4, 128>();          // bins complete
          const int64_t ray = item * 2 + rr;
          const float* wr = fz->w + rr * FS;
          const float* uu = (a.u && fz->ray[rr][7] != 0.0f) ? a.u + ray * FI : nullptr;
          if (t64 < 32) ray_build_cdf([&](int k) { return wr[k + 1]; }, FS - 1, fz->cdf[rr], t64);
          named_bar_sync<4, 128>();
          for (int sidx = t64; sidx < FI; sidx += 64)
            fz->vals[rr][FS + sidx] = ray_sample_at(fz->bins[rr], fz->cdf[rr], FS - 1, uu ? uu[sidx] : linspace01(sidx, FI));
          named_bar_sync<4, 128>();
          // both runs ascending (always, for the deterministic linspace)?  One vote for the pair keeps the barrier simple.
          const bool mine = (uu == nullptr) && ray_sorted_part(fz->vals[rr] + FS, FI, t64, 64) && ray_sorted_part(fz->vals[rr], FS, t64, 64);
          int all_sorted;
          __syncwarp();
          asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.s32 p, %1, 0;\n\tbarrier.red.and.pred q, 4, 128, p;\n\tselp.s32 %0, 1, 0, q;\n\t}"
                       : "=r"(all_sorted) : "r"((int)mine) : "memory");
          if (all_sorted) ray_merge_part(fz->vals[rr], FS, fz->vals[rr] + FS, FI, fz->zf[rr], t64, 64);
          else ray_rank_part(fz->vals[rr], FF, fz->zf[rr], t64, 64);
          named_bar_sync<4, 128>();
          if (a.zf_out && fz->ray[rr][7] != 0.0f)
            for (int k = t64; k < FF; k += 64) a.zf_out[ray * FF + k] = fz->zf[rr][k];
        }
      }
      all_sync();                        // the logits region is free again; fine depths visible to the next prologue
    }
  }
}

// ------------------------------------------------------------------------------------------------ host: program
static void build_program(Program& P, int ins_num) {
  memset(&P, 0, sizeof(P));
  P.ins_num = ins_num;
  // Slot 0 always holds K-half 0 of the current activation, slot 1 K-half 1 (see the MMA role of the kernel).
  int a_step = -1, b_step = -1;                        // steps that produced them
  int t = 0;
  auto add_chunk = [&](Step& s, int kind, int dep, int ks) {
    s.chunk[s.n_chunks] = (int8_t)kind; s.dep[s.n_chunks] = (int8_t)dep; s.ksteps[s.n_chunks] = (int8_t)ks; ++s.n_chunks;
  };
  auto add_act = [&](Step& s) {
    add_chunk(s, 0, a_step, 4); add_chunk(s, 1, a_step, 4);
    add_chunk(s, 2, b_step, 4); add_chunk(s, 3, b_step, 4);
  };
  for (int l = 0; l < 8; ++l) {
    for (int h = 0; h < 2; ++h) {
      Step& s = P.step[t];
      s.n = 128; s.relu = 1; s.out_slot = (int8_t)h;
      if (l == 0) add_chunk(s, CK_E, -1, 4);
      else { add_act(s); if (l == 5) add_chunk(s, CK_E, -1, 4); }
      ++t;
    }
    a_step = t - 2; b_step = t - 1;
  }
  // folded instance branch -> slot 0; folded colour branch (its 3-wide head runs on CUDA cores); instance head on slot 0
  { Step& s = P.step[t]; s.n = 128; s.relu = 1; s.out_slot = 0; add_act(s); ++t; }                              // T_INS_HID
  { Step& s = P.step[t]; s.n = 128; s.relu = 1; s.out_slot = -1; add_act(s); add_chunk(s, CK_D, -1, 2); ++t; }  // T_RGB_HID
  { Step& s = P.step[t]; s.n = (int16_t)(((ins_num + 1) + 15) / 16 * 16); s.relu = 0; s.out_slot = -1;        // T_INS_OUT
    add_chunk(s, 0, t - 2, 4); add_chunk(s, 1, t - 2, 4); ++t; }
  // stage offsets
  uint32_t off = 0;
  int si = 0;
  for (int i = 0; i < N_STEPS; ++i)
    for (int c = 0; c < 2 * P.step[i].n_chunks; ++c) { P.stage_off[si++] = off; off += (uint32_t)P.step[i].n * 128u; }
  P.stage_off[si] = off;               // sentinel: total image size
  P.n_stages = si;
}

// ------------------------------------------------------------------------------------------------ host: packing
struct PackStage {            // one entry per (step, chunk): produces the W_hi and the W_lo stage
  const float* src; int ld; int n_base; int n_valid; int col_base; int k_valid; int n_rows; uint32_t off_hi; uint32_t off_lo;
  int transposed;             // 0: B[n][k] = src[n_base + n][col_base + k];  1: B[n][k] = src[col_base + k][n_base + n]
};

__global__ void fold_kernel(const float* __restrict__ w2, int ld2, const float* __restrict__ w1, const float* __restrict__ b1,
                            const float* __restrict__ b2, int extra_cols, float* __restrict__ wout, float* __restrict__ bout) {
  // wout[n][k] = sum_j w2[n][j] w1[j][k] (k < 256);  wout[n][256 + e] = w2[n][256 + e];  bout[n] = sum_j w2[n][j] b1[j] + b2[n]
  // grid (128 output rows, column blocks): FOUR lanes per output element, each with a 64-long fp64 chain, combined by shuffles
  // (this kernel is on the critical path of every training step: the weights change, the fold is redone)
  const int n = blockIdx.x, ldo = 256 + extra_cols, sub = threadIdx.x & 3;
  const int per_block = blockDim.x >> 2;
  for (int k0 = blockIdx.y * per_block; k0 < ldo + 1; k0 += gridDim.y * per_block) {
    const int k = k0 + (threadIdx.x >> 2);
    double s = 0.0;
    if (k < 256) {
      for (int j = sub * 64; j < sub * 64 + 64; ++j) s += (double)w2[(size_t)n * ld2 + j] * (double)w1[(size_t)j * 256 + k];
    } else if (k == ldo) {
      for (int j = sub * 64; j < sub * 64 + 64; ++j) s += (double)w2[(size_t)n * ld2 + j] * (double)b1[j];
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    if (sub != 0 || k > ldo) continue;
    if (k < 256) wout[(size_t)n * ldo + k] = (float)s;
    else if (k < ldo) wout[(size_t)n * ldo + k] = w2[(size_t)n * ld2 + k];
    else bout[n] = (float)(s + (double)b2[n]);
  }
}

__global__ void pack_kernel(const PackStage* __restrict__ stages, int n_entries, uint8_t* __restrict__ image) {
  const int e = blockIdx.x;
  if (e >= n_entries) return;
  const PackStage ps = stages[e];
  for (int idx = threadIdx.x; idx < ps.n_rows * 8; idx += blockDim.x) {
    const int n = idx >> 3, u = idx & 7;
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = 8 * u + 2 * j + h;
        v[h] = !(n < ps.n_valid && k < ps.k_valid) ? 0.0f
               : (ps.transposed ? ps.src[(size_t)(ps.col_base + k) * ps.ld + ps.n_base + n]
                                : ps.src[(size_t)(ps.n_base + n) * ps.ld + ps.col_base + k]);
      }
      umma::split_bf16x2(v[0], v[1], hi[j], lo[j]);
    }
    const uint32_t o = umma::sw128_offset(n, 8 * u);
    *reinterpret_cast<uint4*>(image + ps.off_hi + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(image + ps.off_lo + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

__global__ void bias_kernel(NetParams p, const float* __restrict__ fold_b_rgb, const float* __restrict__ fold_b_ins,
                            float* __restrict__ bias) {
  // [N_STEPS][128] step biases, then the CUDA-core layers: density weights / bias, rgb_linear weights / bias (B_* offsets)
  for (int i = threadIdx.x + blockIdx.x * blockDim.x; i < B_TOTAL; i += blockDim.x * gridDim.x) {
    float v = 0.0f;
    if (i < 16 * 128) {
      const int t = i / 128, c = i % 128, l = t / 2, h = t % 2;
      v = p.b[l][h * 128 + c];
    } else if (i < (T_INS_HID + 1) * 128) v = fold_b_ins[i - T_INS_HID * 128];
    else if (i < (T_RGB_HID + 1) * 128) v = fold_b_rgb[i - T_RGB_HID * 128];
    else if (i < (T_INS_OUT + 1) * 128) { const int c = i - T_INS_OUT * 128; v = c < p.ins_num + 1 ? p.b[L_INS_OUT][c] : 0.0f; }
    else if (i < B_WD + 256) v = p.w[L_DENSITY][i - B_WD];
    else if (i == B_BD) v = p.b[L_DENSITY][0];
    else if (i >= B_WRGB && i < B_WRGB + 3 * 128) v = p.w[L_RGB_OUT][i - B_WRGB];
    else if (i >= B_BRGB && i < B_BRGB + 3) v = p.b[L_RGB_OUT][i - B_BRGB];
    bias[i] = v;
  }
}

}  // namespace uk

// ================================================================================================ API
struct UmmaExtra {            // hangs off UmmaWeights::image allocation bookkeeping
  uk::Program prog;
  float* fold_w_rgb; float* fold_w_ins; float* fold_b; uk::PackStage* d_entries;
  int32_t* d_status;          // device alias of h_status
  volatile int32_t* h_status;  // error word in mapped host memory: a kernel that gave up on a barrier writes its code here, and the
                              // NEXT launch through this weight set refuses to start (a stalled launch can never pass silently)
};

static UmmaExtra* extra_of(const UmmaWeights& w) { return reinterpret_cast<UmmaExtra*>(w.extra); }

void umma_weights_free(UmmaWeights& w) {
  if (w.image) cudaFree(w.image);
  if (w.bias) cudaFree(w.bias);
  if (w.extra) {
    UmmaExtra* x = extra_of(w);
    if (x->fold_w_rgb) cudaFree(x->fold_w_rgb);
    if (x->fold_w_ins) cudaFree(x->fold_w_ins);
    if (x->fold_b) cudaFree(x->fold_b);
    if (x->d_entries) cudaFree(x->d_entries);
    if (x->h_status) cudaFreeHost((void*)x->h_status);
    delete x;
  }
  w = UmmaWeights();
}

bool umma_available(const UmmaWeights& w) { return w.ready; }
const float* umma_fold_w_rgb(const UmmaWeights& w) { return w.extra ? extra_of(w)->fold_w_rgb : nullptr; }
int32_t* umma_status_word(const UmmaWeights& w) { return w.extra ? extra_of(w)->d_status : nullptr; }
int umma_status_peek(const UmmaWeights& w) { return (w.extra && extra_of(w)->h_status) ? (int)*extra_of(w)->h_status : 0; }

int umma_weights_pack(UmmaWeights& w, const NetParams& p, cudaStream_t st) {
  using namespace uk;
  if (w.extra && w.ins_num != p.ins_num) umma_weights_free(w);
  if (!w.extra) {
    UmmaExtra* x = new UmmaExtra();
    memset(x, 0, sizeof(*x));
    build_program(x->prog, p.ins_num);
    w.extra = x;
    w.ins_num = p.ins_num;
    w.image_bytes = x->prog.stage_off[x->prog.n_stages];
    DMN_CUDA(cudaMalloc(&w.image, w.image_bytes));
    DMN_CUDA(cudaMalloc((void**)&w.bias, B_TOTAL * sizeof(float)));
    DMN_CUDA(cudaMalloc((void**)&x->fold_w_rgb, 128 * 283 * sizeof(float)));
    DMN_CUDA(cudaMalloc((void**)&x->fold_w_ins, 128 * 256 * sizeof(float)));
    DMN_CUDA(cudaMalloc((void**)&x->fold_b, 256 * sizeof(float)));
    DMN_CUDA(cudaMalloc((void**)&x->d_entries, MAX_STAGES * sizeof(PackStage)));
    DMN_CUDA(cudaHostAlloc((void**)&x->h_status, sizeof(int32_t), cudaHostAllocMapped));
    *x->h_status = 0;
    DMN_CUDA(cudaHostGetDevicePointer((void**)&x->d_status, (void*)x->h_status, 0));
  }
  UmmaExtra* x = extra_of(w);
  // fold the activation-free feature layers into the following hidden layers (fp64 accumulate)
  fold_kernel<<<dim3(128, 5), 256, 0, st>>>(p.w[L_RGB_HID], 283, p.w[L_RGB_FEAT], p.b[L_RGB_FEAT], p.b[L_RGB_HID], 27, x->fold_w_rgb, x->fold_b);
  DMN_LAUNCH_OK();
  fold_kernel<<<dim3(128, 5), 256, 0, st>>>(p.w[L_INS_HID], 256, p.w[L_INS_FEAT], p.b[L_INS_FEAT], p.b[L_INS_HID], 0, x->fold_w_ins, x->fold_b + 128);
  DMN_LAUNCH_OK();
  // one PackStage per (step, chunk)
  std::vector<PackStage> ent;
  int si = 0;
  for (int t = 0; t < N_STEPS; ++t) {
    const Step& s = x->prog.step[t];
    for (int c = 0; c < s.n_chunks; ++c, si += 2) {
      PackStage e;
      memset(&e, 0, sizeof(e));
      e.n_rows = s.n; e.off_hi = x->prog.stage_off[si]; e.off_lo = x->prog.stage_off[si + 1];
      const int kind = s.chunk[c];
      if (t < 16) {                                   // trunk layer l, output half h
        const int l = t / 2, h = t % 2;
        e.src = p.w[l]; e.ld = layer_in(l); e.n_base = h * 128; e.n_valid = 128;
        if (kind == CK_E) { e.col_base = (l == 0) ? 0 : 256; e.k_valid = 63; }
        else { e.col_base = 64 * c; e.k_valid = 64; }
      } else if (t == T_RGB_HID) {                    // folded rgb hidden layer: [128][283]
        e.src = x->fold_w_rgb; e.ld = 283; e.n_base = 0; e.n_valid = 128;
        if (kind == CK_D) { e.col_base = 256; e.k_valid = 27; } else { e.col_base = 64 * c; e.k_valid = 64; }
      } else if (t == T_INS_HID) {                    // folded instance hidden layer: [128][256]
        e.src = x->fold_w_ins; e.ld = 256; e.n_base = 0; e.n_valid = 128; e.col_base = 64 * c; e.k_valid = 64;
      } else {                                        // ins_linear [ins_num+1][128]
        e.src = p.w[L_INS_OUT]; e.ld = 128; e.n_base = 0; e.n_valid = p.ins_num + 1; e.col_base = 64 * c; e.k_valid = 64;
      }
      ent.push_back(e);
    }
  }
  DMN_CHECK((int)ent.size() * 2 == x->prog.n_stages && (int)ent.size() <= MAX_STAGES, "umma pack: stage table mismatch");
  const size_t n_fwd = ent.size();
  DMN_CUDA(cudaMemcpyAsync(x->d_entries, ent.data(), ent.size() * sizeof(PackStage), cudaMemcpyHostToDevice, st));
  DMN_CUDA(cudaStreamSynchronize(st));               // `ent` is a host temporary
  pack_kernel<<<(unsigned)n_fwd, 256, 0, st>>>(x->d_entries, (int)n_fwd, (uint8_t*)w.image);
  DMN_LAUNCH_OK();
  bias_kernel<<<8, 256, 0, st>>>(p, x->fold_b, x->fold_b + 128, w.bias);
  DMN_LAUNCH_OK();
  w.ready = true;
  return 0;
}

int launch_mlp_umma(const UmmaWeights& w, const NetParams& p, const float* x, const float* rays_o, const float* rays_d,
                    const float* z, int64_t m, int s, float* out, float* acts, cudaStream_t st) {
  using namespace uk;
  DMN_CHECK(w.ready && w.extra, "mlp(umma): weights not packed (call dmnerf_set_weights first)");
  DMN_CHECK((x != nullptr) != (rays_o != nullptr && rays_d != nullptr), "mlp(umma): pass either x or rays");
  DMN_CHECK(x != nullptr || z != nullptr || s == 1, "mlp(umma): points mode (z == NULL) takes one sample per row");
  DMN_CHECK(umma_status_peek(w) == 0, "mlp(umma): an earlier tensor-core launch reported protocol error %d (bounded wait expired); its results "
            "are invalid -- destroy the context", umma_status_peek(w));
  if (m == 0) return 0;
  UmmaExtra* ex = extra_of(w);
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    DMN_CUDA(cudaFuncSetAttribute(mlp_umma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  }
  int dev = 0, sms = 0;
  DMN_CUDA(cudaGetDevice(&dev));
  DMN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int64_t tiles = (m + TILE_M - 1) / TILE_M;
  KArgs a;
  memset(&a, 0, sizeof(a));
  a.image = (const uint8_t*)w.image; a.bias = w.bias; a.x = x; a.rays_o = rays_o; a.rays_d = rays_d; a.z = z;
  a.m = m; a.s = s; a.out = out; a.acts = acts; a.status = ex->d_status;
  const unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
  mlp_umma_kernel<false><<<grid, N_THREADS, SMEM_BYTES, st>>>(ex->prog, a);
  DMN_LAUNCH_OK();
  return 0;
}

// Whole dm_nerf() pipeline (render.py:31-96) in ONE launch: coarse network -> composite -> importance sampling -> fine
// network -> composite, per pair of rays, nothing but rays in and per-ray maps out crossing HBM.  64 + 128 samples only.
int launch_render_umma(const UmmaWeights& wc, const UmmaWeights& wf, const dmnerf_render_io* io, int64_t n, int flags,
                       cudaStream_t st) {
  using namespace uk;
  DMN_CHECK(wc.ready && wf.ready && wc.extra && wf.extra, "render(umma): weights not packed");
  DMN_CHECK(wc.ins_num == wf.ins_num, "render(umma): coarse/fine ins_num differ");
  DMN_CHECK(umma_status_peek(wc) == 0, "render(umma): an earlier tensor-core launch reported protocol error %d (bounded wait expired); its "
            "results are invalid -- destroy the context", umma_status_peek(wc));
  if (n == 0) return 0;
  UmmaExtra* ex = extra_of(wc);
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    DMN_CUDA(cudaFuncSetAttribute(mlp_umma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  }
  int dev = 0, sms = 0;
  DMN_CUDA(cudaGetDevice(&dev));
  DMN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  KArgs a;
  memset(&a, 0, sizeof(a));
  a.image = (const uint8_t*)wc.image; a.bias = wc.bias;
  a.image_fine = (const uint8_t*)wf.image; a.bias_fine = wf.bias;
  a.rays_o = io->rays_o; a.rays_d = io->rays_d;
  a.z_in = io->z_coarse; a.z_stride = io->z_row_stride;
  const bool perturb = (flags & DMNERF_FLAG_PERTURB) != 0;
  a.t_rand = perturb ? io->t_rand : nullptr; a.u = perturb ? io->u : nullptr;
  a.n_rays = n; a.keep_all_ins = (flags & DMNERF_FLAG_KEEP_INS) ? 1 : 0;
  a.rgb_c = io->rgb_coarse; a.rgb_f = io->rgb_fine; a.depth_c = io->depth_coarse; a.depth_f = io->depth_fine;
  a.acc_c = io->acc_coarse; a.acc_f = io->acc_fine; a.ins_c = io->ins_coarse; a.ins_f = io->ins_fine;
  a.zc_out = io->z_vals_coarse; a.zf_out = io->z_vals_fine; a.wc_out = io->weights_coarse; a.wf_out = io->weights_fine;
  a.status = ex->d_status;
  const int64_t units = (n + 1) / 2;
  const unsigned grid = (unsigned)(units < sms ? units : sms);
  mlp_umma_kernel<true><<<grid, N_THREADS, SMEM_BYTES, st>>>(ex->prog, a);
  DMN_LAUNCH_OK();
  return 0;
}

int umma_check_status(const UmmaWeights& w, cudaStream_t st) {
  if (!w.extra) return 0;
  int32_t code = 0;
  DMN_CUDA(cudaStreamSynchronize(st));
  code = (int32_t)*extra_of(w)->h_status;
  DMN_CHECK(code == 0, "tensor-core MLP kernel reported protocol error %d (bounded wait expired)", code);
  return 0;
}

}  // namespace dmnerf
