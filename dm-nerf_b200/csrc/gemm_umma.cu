// Warpgroup-MMA (wgmma) GEMM kernels for the training backward of the DM_NeRF network (networks/dm_nerf.py:80-106
// differentiated, driven by train_dmsr.py:62-64): the two wide GEMM shapes of every layer,
//
//   gemm_nn:  dX[M, 256]  (+)= dY[M, N] * W[N, 256]            (N = 128 or 256; optional ReLU mask from the saved bit planes)
//   gemm_tn:  dW[NA, 256]  +=  dY[M, NA]^T * X[M, 256]          (NA = 128 or 256; contraction over the M samples)
//
// with the same fp32-grade arithmetic as the forward kernel: every fp32 operand is split into bf16 hi + bf16 lo and each
// product is issued as three tensor passes  A_hi*B_hi + A_lo*B_hi + A_hi*B_lo  into fp32 accumulators in registers.
//
// Operands come straight from the row-major fp32 matrices in global memory; the only preparation is the hi/lo split, done by
// the CUDA cores while the block is written into shared memory.  One loader serves every operand, because the memory image
// of a [rows][64 columns] block in the SWIZZLE_128B layout is the same whether the tensor core reads it K-major (rows = M or
// N index, columns = contraction index: dY in gemm_nn) or MN-major (rows = contraction index, columns = M / N index: W in
// gemm_nn, dY and X in gemm_tn) -- only the descriptor and the transpose flag of the instruction differ.
//
// Structure (both kernels): persistent CTAs, two shared-memory stages.  Every thread splits the block it fetched into
// registers one stage earlier and stores it while the tensor core multiplies the previous stage; the global loads of the stage
// after that are in flight at the same time.  Each warpgroup issues the MMAs of its own 64-row slice of the output tile.
#include <cstring>

#include "common.cuh"
#include "umma.cuh"

namespace dmnerf {
namespace tg {

using namespace umma;

constexpr int NOUT = 256;                  // output columns (gemm_nn) / columns of X (gemm_tn)

// One 16-byte unit of a bf16 slab = 8 consecutive fp32 values of one matrix row.
struct Unit { float v[8]; };

// 8 floats of row r (valid below r_end), columns col.. (valid below c_end) of a row-major matrix; zero outside.
__device__ __forceinline__ void load_unit(Unit& u, const float* __restrict__ src, int64_t ld, int64_t r, int64_t r_end, int col,
                                          int c_end, int vec_ok) {
  if (r < r_end && vec_ok && col + 8 <= c_end) {
    const float4* p4 = reinterpret_cast<const float4*>(src + r * ld + col);
    const float4 x = __ldg(p4), y = __ldg(p4 + 1);
    u.v[0] = x.x; u.v[1] = x.y; u.v[2] = x.z; u.v[3] = x.w; u.v[4] = y.x; u.v[5] = y.y; u.v[6] = y.z; u.v[7] = y.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) u.v[i] = (r < r_end && col + i < c_end) ? __ldg(src + r * ld + col + i) : 0.0f;
  }
}

// The same 8 values of a COLUMN-major matrix (element (r, c) at src[c * col_stride + r]): the embedded-input plane of the
// training forward is stored that way (ActPlanes::emb) so that its writers are coalesced.
__device__ __forceinline__ void load_unit_cm(Unit& u, const float* __restrict__ src, int64_t col_stride, int64_t r, int64_t r_end, int col,
                                             int c_end) {
#pragma unroll
  for (int i = 0; i < 8; ++i) u.v[i] = (r < r_end && col + i < c_end) ? __ldg(src + (int64_t)(col + i) * col_stride + r) : 0.0f;
}

// Split the unit into bf16 hi / lo and store it at (row, 16-byte unit cu) of the two swizzled slabs.
__device__ __forceinline__ void store_unit(const Unit& u, uint8_t* hi, uint8_t* lo, int row, int cu) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_bf16x2(u.v[2 * i], u.v[2 * i + 1], h[i], l[i]);
  const uint32_t o = sw128_offset(row, cu * 8);
  *reinterpret_cast<uint4*>(hi + o) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo + o) = make_uint4(l[0], l[1], l[2], l[3]);
}

__device__ __forceinline__ void fail(int32_t* status, int code) { atomicCAS(status, 0, code); }

// ------------------------------------------------------------------------------------------------ gemm_nn
// C[M, 256] (+)= A[M, N] * W[N, 256]   (dX = dY W; W rows are the contraction index), N = 64 * NCH.
// The weight matrix is the same for every tile, so it is split ONCE per call into a packed image of ready-made stage blocks (pack_w_kernel) that are streamed into the stages with bulk async copies (TMA engine, mbarrier transaction
// counts, requested as soon as a stage is free); the threads only handle the activation / gradient rows.
// Output tile [128 x 256]: warpgroup w owns rows 64 (w & 1) and columns 128 (w >> 1).
constexpr int NN_THREADS = 512;
constexpr uint32_t NN_A_BYTES = 128 * 128;               // one [128 x 64] slab
constexpr uint32_t NN_W_BYTES = 256 * 128;               // the W block of a chunk: 4 slabs [64 x 64]
constexpr uint32_t NN_W_SLAB = 64 * 128;
constexpr uint32_t NN_STAGE = 2 * NN_A_BYTES + 2 * NN_W_BYTES;          // A hi, A lo, W hi, W lo = 96 KB
constexpr uint32_t NN_SMEM = 2 * NN_STAGE + 1024;
constexpr int NN_UA = 128 * 8 / NN_THREADS;              // A units per thread and stage: 2

// image[c] = { W_hi block, W_lo block } of contraction chunk c, in the shared-memory layout of a stage.
__global__ void pack_w_kernel(const float* __restrict__ W, int ldw, int nch, int vec_w, uint8_t* __restrict__ image) {
  const int c = blockIdx.x;
  uint8_t* w_hi = image + (size_t)c * 2 * NN_W_BYTES;
  uint8_t* w_lo = w_hi + NN_W_BYTES;
  for (int u = threadIdx.x; u < 256 * 8; u += blockDim.x) {
    Unit r;
    load_unit(r, W, ldw, 64 * c + ((u >> 3) & 63), 64 * nch, 64 * (u >> 9) + (u & 7) * 8, NOUT, vec_w != 0);
    store_unit(r, w_hi + (u >> 9) * NN_W_SLAB, w_lo + (u >> 9) * NN_W_SLAB, (u >> 3) & 63, u & 7);
  }
}

// mask (fp32 ReLU mask sharing ldc) and bias are always NULL: without these two branches nvcc schedules the epilogue so that
// the accumulating N = 128 launch of the gradient chain takes twice as long (H100 80GB HBM3 at 700 W: 264 -> 515 us per call
// at M = 196608), which outweighs the 5 % the N = 256 launches gain.  Keep them until the epilogue is restructured.
template <int NCH>
__global__ void __launch_bounds__(NN_THREADS, 1) gemm_nn_tc_kernel(const float* __restrict__ A, int lda, const uint8_t* __restrict__ wimage,
                                                                   float* __restrict__ C, int ldc, int64_t M, int accumulate,
                                                                   const float* __restrict__ mask, const uint16_t* __restrict__ mbits,
                                                                   const float* __restrict__ bias, int vec_a, int32_t* status) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ uint64_t wfull[2];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, wg = tid >> 7, wl = (tid >> 5) & 3, lane = tid & 31;
  const int64_t n_tiles = (M + 127) / 128;
  const int64_t my_tiles = (n_tiles > blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const int64_t n_chunks = my_tiles * NCH;
  // chunk q of this CTA: tile blockIdx.x + (q / NCH) * gridDim.x, contraction columns [64 (q % NCH), +64)
  auto request_w = [&](int64_t q) {
    const uint32_t s = (uint32_t)q & 1;
    uint8_t* w_hi = smem + s * NN_STAGE + 2 * NN_A_BYTES;
    const int c = (int)(q % NCH);
    mbar_arrive_expect_tx(&wfull[s], 2 * NN_W_BYTES);
#pragma unroll
    for (int i = 0; i < 4; ++i) bulk_g2s(w_hi + i * 16384, wimage + (size_t)c * 2 * NN_W_BYTES + i * 16384, 16384, &wfull[s]);
  };
  if (tid == 0) {
    mbar_init(&wfull[0], 1); mbar_init(&wfull[1], 1);
    fence_barrier_init();
    if (n_chunks > 0) request_w(0);
    if (n_chunks > 1) request_w(1);
  }
  __syncthreads();
  auto load = [&](Unit (&r)[NN_UA], int64_t q) {
    const int c = (int)(q % NCH);
    const int64_t m0 = (blockIdx.x + (q / NCH) * gridDim.x) * 128;
#pragma unroll
    for (int i = 0; i < NN_UA; ++i) {
      const int u = tid + i * NN_THREADS;
      load_unit(r[i], A, lda, m0 + (u >> 3), M, 64 * c + (u & 7) * 8, 64 * NCH, vec_a != 0);
    }
  };
  auto store = [&](const Unit (&r)[NN_UA], int64_t q) {
    uint8_t* st = smem + ((uint32_t)q & 1) * NN_STAGE;
#pragma unroll
    for (int i = 0; i < NN_UA; ++i) {
      const int u = tid + i * NN_THREADS;
      store_unit(r[i], st, st + NN_A_BYTES, u >> 3, u & 7);
    }
  };
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
  Unit r[NN_UA];
  if (n_chunks > 0) { load(r, 0); store(r, 0); }
  if (n_chunks > 1) load(r, 1);
  for (int64_t q = 0; q < n_chunks; ++q) {
    const int c = (int)(q % NCH);
    const int64_t ti = q / NCH;
    const uint32_t s = (uint32_t)q & 1;
    fence_proxy_async_smem();
    __syncthreads();                               // A(q) stored; every warpgroup has finished the MMAs of chunk q - 1
    if (tid == 0 && q >= 1 && q + 1 < n_chunks) request_w(q + 1);     // into the stage chunk q - 1 used
    if (!mbar_wait(&wfull[s], (uint32_t)(q >> 1) & 1)) fail(status, 604);
    {
      const uint32_t st = smem_u32(smem + s * NN_STAGE);
      const uint32_t sa_hi = st + (wg & 1) * 8192, sa_lo = sa_hi + NN_A_BYTES;
      const uint32_t sw_hi = st + 2 * NN_A_BYTES + (wg >> 1) * 16384, sw_lo = sw_hi + NN_W_BYTES;
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t da_hi = make_sdesc_sw128(sa_hi + ks * 32), da_lo = make_sdesc_sw128(sa_lo + ks * 32);
        const uint64_t db_hi = sdesc(sw_hi + ks * 2048, NN_W_SLAB, 1024);
        const uint64_t db_lo = sdesc(sw_lo + ks * 2048, NN_W_SLAB, 1024);
        wgmma_n128<0, 1>(acc, da_hi, db_hi, (c == 0 && ks == 0) ? 0u : 1u);
        wgmma_n128<0, 1>(acc, da_lo, db_hi, 1u);
        wgmma_n128<0, 1>(acc, da_hi, db_lo, 1u);
      }
      wg_commit();
    }
    if (q + 1 < n_chunks) store(r, q + 1);          // split the next block while the tensor core works on this one
    if (q + 2 < n_chunks) load(r, q + 2);
    wg_wait<0>();
    wg_reg_fence(acc);
    if (c == NCH - 1) {
      // epilogue: thread -> rows m0 + 64 (wg & 1) + 16 wl + lane / 4 (+ 8), columns 128 (wg >> 1) + 8 j + 2 (lane % 4) (+ 1)
      const int64_t m_a = (blockIdx.x + ti * gridDim.x) * 128 + 64 * (wg & 1) + 16 * wl + (lane >> 2);
      const int col0 = 128 * (wg >> 1) + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t m = m_a + 8 * h;
        if (m >= M) continue;
        float* crow = C + m * ldc;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = col0 + 8 * j;
          float2 o = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          if (bias) { const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col)); o.x += bb.x; o.y += bb.y; }
          if (accumulate) { const float2 old = *reinterpret_cast<const float2*>(crow + col); o.x += old.x; o.y += old.y; }
          if (mask) {
            const float2 mk = __ldg(reinterpret_cast<const float2*>(mask + m * ldc + col));
            if (!(mk.x > 0.0f)) o.x = 0.0f;
            if (!(mk.y > 0.0f)) o.y = 0.0f;
          }
          if (mbits) {                   // 1-bit ReLU mask: [16 groups][M] uint16, bit c of group g = unit 16 g + c
            const uint32_t b = (uint32_t)__ldg(mbits + (int64_t)(col >> 4) * M + m) >> (col & 15);
            if (!(b & 1u)) o.x = 0.0f;
            if (!(b & 2u)) o.y = 0.0f;
          }
          *reinterpret_cast<float2*>(crow + col) = o;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ gemm_tn
// P[NA, NB] = A[mb:me, 0:NA]^T * B[mb:me, 0:nb] for this CTA's rows; the CTA computes one [128 x NBT] tile of P (NBT = 64 with
// NB = 64, else 128; columns from nb on are zero) over 32 samples per stage.  Both operands are MN-major (the samples are the
// contraction index).
// Every CTA writes its partial product to its own slice of a scratch buffer; reduce_partials_kernel adds the slices into the
// gradient in a fixed order.  colsum != NULL: colsum[n] += sum over the rows of A[:, n] (the bias gradient, from the registers
// that already hold A); each CTA sums its rows in a fixed order into one row of column sums per slice, which
// reduce_partials_kernel adds in slice order like the products.
constexpr int TN_THREADS = 256;
constexpr uint32_t TN_SLAB = 32 * 128;                   // one [32 samples x 64 columns] block
constexpr int64_t TN_MAX_ROWS = 16384;                   // samples per slice at most (launch_gemm_tn_tc_batch)

// A launch multiplies up to TN_MAX_BATCH independent products over the same M samples (the weight gradients of several layers of
// one network: their operands are all on hand once the gradient chain has run).  blockIdx.x = ((prob * tiles) + tile) * slices + slice.
struct TnBatch {
  TnProblem p[TN_MAX_BATCH];
  int vec_a[TN_MAX_BATCH], vec_b[TN_MAX_BATCH];
  int n, slices;
  int64_t rows_per_cta;
};

template <int NBT>
__global__ void __launch_bounds__(TN_THREADS, 1) gemm_tn_tc_kernel(const __grid_constant__ TnBatch batch, float* __restrict__ partial,
                                                                   int64_t M, int NA, int NB, int32_t* status) {
  constexpr int SB = NBT / 64;                           // B blocks per stage
  constexpr uint32_t STAGE = 2 * (2 + SB) * TN_SLAB;     // A (2 blocks) + B, hi + lo
  constexpr int UPT = ((2 + SB) * 256) / TN_THREADS;     // units per thread per stage: unit U = tid + i * TN_THREADS
  constexpr int NACC = NBT / 2;
  const int tiles_n = NA / 128, tiles_k = NB / NBT, tiles = tiles_n * tiles_k;
  const int slice = (int)blockIdx.x % batch.slices, pt = (int)blockIdx.x / batch.slices;
  const int prob = pt / tiles, tile = pt % tiles, tn = tile / tiles_k, tk = tile % tiles_k;
  const float* __restrict__ A = batch.p[prob].A;
  const float* __restrict__ B = batch.p[prob].B;
  float* __restrict__ colsum = tk == 0 ? batch.p[prob].colsum : nullptr;
  const int lda = batch.p[prob].lda, ldb = batch.p[prob].ldb, nb = batch.p[prob].K;
  const int vec_a = batch.vec_a[prob], vec_b = batch.vec_b[prob];
  const int64_t b_cm = batch.p[prob].b_cm, rows_per_cta = batch.rows_per_cta;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ float csum_s[32][128];                      // [row of a stage][column]: the per-thread column sums
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, wg = tid >> 7, wl = (tid >> 5) & 3, lane = tid & 31;
  const int64_t mb = (int64_t)slice * rows_per_cta;
  const int64_t me = (mb + rows_per_cta < M) ? mb + rows_per_cta : M;
  const int64_t n_chunks = (me > mb) ? (me - mb + 31) / 32 : 0;
  float csum[UPT][8];
#pragma unroll
  for (int i = 0; i < UPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) csum[i][j] = 0.0f;
  auto load = [&](Unit (&r)[UPT], int64_t q) {
    const int64_t m0 = mb + q * 32;
#pragma unroll
    for (int i = 0; i < UPT; ++i) {
      const int U = tid + i * TN_THREADS, blk = U >> 8, u = U & 255;
      if (blk < 2) load_unit(r[i], A, lda, m0 + (u >> 3), me, 128 * tn + 64 * blk + (u & 7) * 8, NA, vec_a);
      else if (b_cm) load_unit_cm(r[i], B, b_cm, m0 + (u >> 3), me, NBT * tk + 64 * (blk - 2) + (u & 7) * 8, nb);
      else load_unit(r[i], B, ldb, m0 + (u >> 3), me, NBT * tk + 64 * (blk - 2) + (u & 7) * 8, nb, vec_b);
    }
  };
  auto store = [&](const Unit (&r)[UPT], int64_t q) {
    uint8_t* st = smem + ((uint32_t)q & 1) * STAGE;
#pragma unroll
    for (int i = 0; i < UPT; ++i) {
      const int U = tid + i * TN_THREADS, blk = U >> 8, u = U & 255;
      const int side = blk < 2 ? 0 : 1, b = blk < 2 ? blk : blk - 2;
      uint8_t* hi = st + (side ? 2 * 2 * TN_SLAB : 0) + b * TN_SLAB;
      uint8_t* lo = hi + (side ? SB : 2) * TN_SLAB;
      store_unit(r[i], hi, lo, u >> 3, u & 7);
      if (colsum && blk < 2) {
#pragma unroll
        for (int j = 0; j < 8; ++j) csum[i][j] += r[i].v[j];
      }
    }
  };
  float acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.0f;
  Unit r[UPT];
  if (n_chunks > 0) { load(r, 0); store(r, 0); }
  if (n_chunks > 1) load(r, 1);
  for (int64_t q = 0; q < n_chunks; ++q) {
    const uint32_t st = smem_u32(smem + ((uint32_t)q & 1) * STAGE);
    fence_proxy_async_smem();
    __syncthreads();                     // chunk q stored; every warpgroup has finished the MMAs of chunk q - 1
    const uint32_t a_hi = st + wg * TN_SLAB, a_lo = a_hi + 2 * TN_SLAB;
    const uint32_t b_hi = st + 4 * TN_SLAB, b_lo = b_hi + SB * TN_SLAB;
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const uint64_t da_hi = sdesc(a_hi + ks * 2048, TN_SLAB, 1024), da_lo = sdesc(a_lo + ks * 2048, TN_SLAB, 1024);
      const uint64_t db_hi = sdesc(b_hi + ks * 2048, TN_SLAB, 1024), db_lo = sdesc(b_lo + ks * 2048, TN_SLAB, 1024);
      const uint32_t sc = (q == 0 && ks == 0) ? 0u : 1u;
      if constexpr (NBT == 128) {
        wgmma_n128<1, 1>(acc, da_hi, db_hi, sc); wgmma_n128<1, 1>(acc, da_lo, db_hi, 1u); wgmma_n128<1, 1>(acc, da_hi, db_lo, 1u);
      } else {
        wgmma_n64<1, 1>(acc, da_hi, db_hi, sc); wgmma_n64<1, 1>(acc, da_lo, db_hi, 1u); wgmma_n64<1, 1>(acc, da_hi, db_lo, 1u);
      }
    }
    wg_commit();
    if (q + 1 < n_chunks) store(r, q + 1);
    if (q + 2 < n_chunks) load(r, q + 2);
    wg_wait<0>();
    wg_reg_fence(acc);
  }
  // slice layout (private to this kernel and reduce_partials_kernel): [prob][slice][NA][NB] row-major, then the column sums
  // [prob][slice][NA]
  if (colsum) {       // bias gradient: units i < 2 hold A (blk = i, u = tid): thread tid owns stage row tid / 8 of 8 columns
    static_assert(TN_THREADS == 256, "one A unit per thread and block");
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) csum_s[tid >> 3][64 * i + (tid & 7) * 8 + j] = csum[i][j];
    __syncthreads();
    if (tid < 128) {
      float s = 0.0f;
      for (int r = 0; r < 32; ++r) s += csum_s[r][tid];
      partial[(size_t)batch.n * batch.slices * NA * NB + ((size_t)prob * batch.slices + slice) * NA + 128 * tn + tid] = s;
    }
  }
  float* mine = partial + ((size_t)prob * batch.slices + slice) * NA * NB;
  const int n_a = 128 * tn + 64 * wg + 16 * wl + (lane >> 2);
  const int k0 = NBT * tk + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < NBT / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(mine + (size_t)(n_a + 8 * h) * NB + k0 + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
  (void)status;
}

// C[n, k] += sum_slice partial[prob][slice][n][k]  (k < K valid columns of the NB-wide partials) for product blockIdx.y of the
// batch; transpose: C[k, n] instead (the product was computed with the roles of the two operands exchanged); the NA threads after
// the product's add its column sums into pr.colsum.  The slices of a product are added in a fixed order, and so are the rows
// inside a slice: the gradient is reproducible from run to run, bit for bit.
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ partial, const __grid_constant__ TnBatch batch,
                                                              int NA, int NB) {
  const TnProblem& pr = batch.p[blockIdx.y];
  const int n_cta = batch.slices, kb = pr.K, ldc = pr.ldc, transpose = pr.transpose;
  float* __restrict__ C = pr.C;
  const int idx4 = blockIdx.x * blockDim.x + threadIdx.x, total4 = NA * NB / 4;
  if (idx4 >= total4) {
    const int n = idx4 - total4;
    if (n >= NA || !pr.colsum) return;
    const float* cs = partial + (size_t)batch.n * n_cta * NA * NB + (size_t)blockIdx.y * n_cta * NA + n;
    float s = 0.0f;
    for (int c = 0; c < n_cta; ++c) s += cs[(size_t)c * NA];
    pr.colsum[n] += s;
    return;
  }
  const float4* src = reinterpret_cast<const float4*>(partial) + (size_t)blockIdx.y * n_cta * total4 + idx4;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = 0; c < n_cta; ++c) {
    const float4 x = __ldcs(src + (size_t)c * total4);
    s.x += x.x; s.y += x.y; s.z += x.z; s.w += x.w;
  }
  const float v[4] = {s.x, s.y, s.z, s.w};
  const int n = (idx4 * 4) / NB, k0 = (idx4 * 4) % NB;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int k = k0 + e;
    if (k >= kb) continue;
    if (transpose) C[(size_t)k * ldc + n] += v[e];
    else C[(size_t)n * ldc + k] += v[e];
  }
}

// rows are 16-byte aligned (128-bit loads)
static int vec4_ok(const void* p, int ld) { return ((uintptr_t)p % 16 == 0) && (ld % 4 == 0); }

}  // namespace tg

// Shapes the dW kernel is specialised for.
bool gemm_tn_tc_supported(int N, int K) { return (N == 128 || N == 256) && (K == 256 || (K >= 1 && K <= 128)); }

// C[M,256] (+)= A[M,N] W[N,256], N = 128 or 256, masked by mask_bits when given.
int launch_gemm_nn_tc(const float* A, int lda, const float* W, int ldw, float* C, int ldc, int64_t M, int N, int accumulate,
                      const uint16_t* mask_bits, DeviceBuffer& wimage_buf, int32_t* status, cudaStream_t st) {
  using namespace tg;
  if (M <= 0) return 0;
  uint8_t* wimage;
  int sms = 0;
  if (wimage_buf.get(4 * 2 * NN_W_BYTES, &wimage) || sm_count(&sms)) return 2;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    DMN_CUDA(cudaFuncSetAttribute(gemm_nn_tc_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)NN_SMEM));
    DMN_CUDA(cudaFuncSetAttribute(gemm_nn_tc_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)NN_SMEM));
  }
  const int64_t tiles = (M + 127) / 128;
  const unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
  const int va = vec4_ok(A, lda), vw = vec4_ok(W, ldw), nch = N / 64;
  pack_w_kernel<<<nch, 512, 0, st>>>(W, ldw, nch, vw, wimage);
  DMN_LAUNCH_OK();
  if (N == 128) gemm_nn_tc_kernel<2><<<grid, NN_THREADS, NN_SMEM, st>>>(A, lda, wimage, C, ldc, M, accumulate, nullptr, mask_bits, nullptr, va, status);
  else gemm_nn_tc_kernel<4><<<grid, NN_THREADS, NN_SMEM, st>>>(A, lda, wimage, C, ldc, M, accumulate, nullptr, mask_bits, nullptr, va, status);
  DMN_LAUNCH_OK();
  return 0;
}

// For every product i < n:  C_i[N, K_i] += A_i[M, N]^T B_i[M, K_i]  (N = 128 or 256; the K_i of one batch are all in one class
// NB: K_i <= 64 -> 64, 65..128 -> 128, 256 -> 256); transpose != 0: the caller passes the WIDE matrix as A and the narrow one
// (K <= 128 columns) as B and wants C[K, N] += B^T A.  One GEMM launch + one reduction launch for the whole batch.
int launch_gemm_tn_tc_batch(const TnProblem* probs, int n, int64_t M, int N, DeviceBuffer& partial, int32_t* status,
                            cudaStream_t st) {
  using namespace tg;
  if (M <= 0 || n <= 0) return 0;
  DMN_CHECK(n <= TN_MAX_BATCH, "gemm_tn(tc): %d products in one batch (max %d)", n, TN_MAX_BATCH);
  auto nb_class = [](int K) { return K <= 64 ? 64 : K <= 128 ? 128 : 256; };
  const int NB = nb_class(probs[0].K);
  TnBatch batch;
  memset(&batch, 0, sizeof(batch));
  for (int i = 0; i < n; ++i) {
    const int K = probs[i].K;
    DMN_CHECK(gemm_tn_tc_supported(N, K) && nb_class(K) == NB, "gemm_tn(tc): shape %d x %d not supported", N, K);
    batch.p[i] = probs[i];
    batch.vec_a[i] = vec4_ok(probs[i].A, probs[i].lda);
    batch.vec_b[i] = vec4_ok(probs[i].B, probs[i].ldb);
  }
  const int NBT = NB == 64 ? 64 : 128;
  const int tiles = (N / 128) * (NB / NBT);
  int sms = 0;
  if (sm_count(&sms)) return 2;
  int slices = sms / (n * tiles);
  if (slices < 1) slices = 1;
  // A CTA sums at most TN_MAX_ROWS samples into its fp32 tensor-core accumulators: the error of that chain grows with its
  // length (H100, 8 products x 4 tiles = 4 slices: relative L2 error of the weight gradients 5.5e-5 at 16 384 samples per
  // slice, 1.9e-4 at 49 152).
  if ((M + slices - 1) / slices > TN_MAX_ROWS) slices = (int)((M + TN_MAX_ROWS - 1) / TN_MAX_ROWS);
  int64_t rows = (M + slices - 1) / slices;
  rows = ((rows + 31) / 32) * 32;
  slices = (int)((M + rows - 1) / rows);
  batch.n = n; batch.slices = slices; batch.rows_per_cta = rows;
  const unsigned grid = (unsigned)(n * tiles * slices);
  float* scratch;
  if (partial.get((size_t)n * slices * N * NB + (size_t)n * slices * N, &scratch)) return 2;      // products, then the column sums
  static PerDeviceOnce attr_once;
  auto smem_of = [](int nbt) { return (uint32_t)(2 * 2 * (2 + nbt / 64) * TN_SLAB + 1024); };
  if (attr_once.first()) {
    DMN_CUDA(cudaFuncSetAttribute(gemm_tn_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_of(128)));
    DMN_CUDA(cudaFuncSetAttribute(gemm_tn_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_of(64)));
  }
  if (NBT == 128) gemm_tn_tc_kernel<128><<<grid, TN_THREADS, smem_of(128), st>>>(batch, scratch, M, N, NB, status);
  else gemm_tn_tc_kernel<64><<<grid, TN_THREADS, smem_of(64), st>>>(batch, scratch, M, N, NB, status);
  DMN_LAUNCH_OK();
  reduce_partials_kernel<<<dim3((N * NB / 4 + N + 255) / 256, n), 256, 0, st>>>(scratch, batch, N, NB);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
