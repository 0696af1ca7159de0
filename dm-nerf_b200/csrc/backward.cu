// Backward of the render path (BASELINE config 4: training step, reference train_dmsr.py:62-64).
//
//   * composite_backward_kernel: d(rgb_map, depth_map, acc_map, ins_map) -> d raw, one warp per ray.  The transmittance
//     product is differentiated in closed form with a reverse warp scan:  dL/dalpha_i = gw_i T_i - (sum_{j>i} gw_j w_j) / f_i.
//     Honours the reference's detach topology (render.py:22-23: the instance map sees detached weights).
//   * MLP backward over the activations saved by the training forward (ActPlanes), with the heads folded like in the forward
//     (mlp_backward_chain): the gradient chain of bwd_chain.cu carries dY through the trunk, batched split-bf16 wgmma GEMMs
//     (gemm_umma.cu) form the weight gradients, small fp32 products give the folded head layers.  Gradient routing is the
//     reference's (dm_nerf.py:95: the instance branch reads h.detach(), so it contributes to ins_feature_linear and below only).

#include "ray_ops.cuh"
#include "umma_api.cuh"

namespace dmnerf {

// ================================================================================================ composite backward
constexpr int CB_WARPS = 4;

__global__ void composite_backward_kernel(const float* __restrict__ raw, const float* __restrict__ z,
                                          const float* __restrict__ rays_d, int64_t n, int S, int C, int keep_all,
                                          const float* __restrict__ g_rgb, const float* __restrict__ g_depth,
                                          const float* __restrict__ g_acc, const float* __restrict__ g_ins,
                                          const float* __restrict__ g_w, float* __restrict__ d_raw, int accumulate) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * CB_WARPS + warp;
  if (ray >= n) return;
  float* w = smem + (size_t)warp * 5 * S;      // weights
  float* T = w + S;                            // exclusive transmittance
  float* fi = T + S;                           // 1 - alpha + 1e-10
  float* ex = fi + S;                          // delta_i * exp(-sigma_i delta_i)  (= d alpha / d sigma)
  float* gw = ex + S;                          // dL/dw_i
  const float* zr = z + ray * S;
  const float* rr = raw + ray * S * C;
  float* dr = d_raw + ray * S * C;
  const float dx = rays_d[ray * 3], dy = rays_d[ray * 3 + 1], dz = rays_d[ray * 3 + 2];
  const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
  const int n_ins_out = keep_all ? C - 4 : C - 5;

  // ---- forward recompute (render.py:7-18) keeping alpha-chain intermediates
  float carry = 1.0f;
  for (int base = 0; base < S; base += 32) {
    const int i = base + lane;
    float alpha = 0.0f, f = 1.0f, dads = 0.0f;
    if (i < S) {
      const float dist = ((i == S - 1) ? 1e10f : zr[i + 1] - zr[i]) * dnorm;
      const float sg = fmaxf(rr[(size_t)i * C + 3], 0.0f);
      const float e = expf(-sg * dist);
      alpha = 1.0f - e;
      f = (1.0f - alpha) + 1e-10f;
      dads = dist * e;
    }
    const float incl = warp_scan_mul(f, lane);
    float excl = __shfl_up_sync(FULL, incl, 1);
    if (lane == 0) excl = 1.0f;
    if (i < S) { T[i] = carry * excl; w[i] = alpha * T[i]; fi[i] = f; ex[i] = dads; }
    carry *= __shfl_sync(FULL, incl, 31);
  }
  __syncwarp();

  // ---- dL/dw_i and the colour-logit gradients
  const float gr0 = g_rgb ? g_rgb[ray * 3] : 0.0f, gr1 = g_rgb ? g_rgb[ray * 3 + 1] : 0.0f, gr2 = g_rgb ? g_rgb[ray * 3 + 2] : 0.0f;
  const float gd = g_depth ? g_depth[ray] : 0.0f, ga = g_acc ? g_acc[ray] : 0.0f;
  for (int i = lane; i < S; i += 32) {
    const float s0 = sigmoidf_acc(rr[(size_t)i * C]), s1 = sigmoidf_acc(rr[(size_t)i * C + 1]), s2 = sigmoidf_acc(rr[(size_t)i * C + 2]);
    gw[i] = gr0 * s0 + gr1 * s1 + gr2 * s2 + gd * zr[i] + ga + (g_w ? g_w[ray * S + i] : 0.0f);
    const float wi = w[i];
    float v0 = gr0 * wi * s0 * (1.0f - s0), v1 = gr1 * wi * s1 * (1.0f - s1), v2 = gr2 * wi * s2 * (1.0f - s2);
    if (accumulate) { v0 += dr[(size_t)i * C]; v1 += dr[(size_t)i * C + 1]; v2 += dr[(size_t)i * C + 2]; }
    dr[(size_t)i * C] = v0; dr[(size_t)i * C + 1] = v1; dr[(size_t)i * C + 2] = v2;
  }
  __syncwarp();

  // ---- instance logits: ins_map_k = sigmoid(sum_i w_i raw_ik); weights are detached unless keep_all (manipulator_render).
  // Lanes run over the samples like in the other phases (the channel index is warp-uniform): every lane owns samples lane,
  // lane + 32, ... -- no serial pass over all S samples per channel, and the keep_all term lands in gw[i] of the owning lane.
  for (int k = 0; k < C - 4; ++k) {
    float a = 0.0f;
    for (int i = lane; i < S; i += 32) a = fmaf(w[i], rr[(size_t)i * C + 4 + k], a);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) a += __shfl_xor_sync(FULL, a, d);
    const float sk = sigmoidf_acc(a);
    const float gk = (g_ins && k < n_ins_out) ? g_ins[ray * n_ins_out + k] * sk * (1.0f - sk) : 0.0f;
    for (int i = lane; i < S; i += 32) {
      float v = gk * w[i];
      if (accumulate) v += dr[(size_t)i * C + 4 + k];
      dr[(size_t)i * C + 4 + k] = v;
      if (keep_all && gk != 0.0f) gw[i] += gk * rr[(size_t)i * C + 4 + k];
    }
  }
  __syncwarp();

  // ---- density: reverse exclusive scan of gw_j w_j, then the closed-form d alpha
  float suffix = 0.0f;                                   // sum over samples after the current chunk
  const int n_chunks = (S + 31) / 32;
  for (int cb = n_chunks - 1; cb >= 0; --cb) {
    const int i = cb * 32 + lane;
    const float p = (i < S) ? gw[i] * w[i] : 0.0f;
    float incl = p;                                      // inclusive suffix sum inside the chunk
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const float o = __shfl_down_sync(FULL, incl, d);
      if (lane + d < 32) incl += o;
    }
    // sum_{j > i} gw_j w_j from the next lane's inclusive sum, not as incl - p: where alpha_i -> 1, p = gw_i w_i is large next
    // to the suffix, and the rounding of that difference would be amplified by 1 / f_i below
    float after = __shfl_down_sync(FULL, incl, 1);
    if (lane == 31) after = 0.0f;
    const float R = suffix + after;
    if (i < S) {
      const float dalpha = gw[i] * T[i] - R / fi[i];
      float v = (rr[(size_t)i * C + 3] > 0.0f) ? dalpha * ex[i] : 0.0f;
      if (accumulate) v += dr[(size_t)i * C + 3];
      dr[(size_t)i * C + 3] = v;
    }
    suffix += __shfl_sync(FULL, incl, 0);
  }
}

int launch_composite_backward(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c, int keep_all,
                              const float* g_rgb, const float* g_depth, const float* g_acc, const float* g_ins,
                              const float* g_weights, float* d_raw, int accumulate, cudaStream_t st) {
  DMN_CHECK(s >= 1 && s <= 2048, "composite_backward: n_samples=%d out of range [1,2048]", s);
  DMN_CHECK(c >= 5 && c <= 4 + DMNERF_MAX_INS + 1, "composite_backward: channels=%d out of range", c);
  if (n == 0) return 0;
  const size_t smem = (size_t)CB_WARPS * 5 * s * sizeof(float);
  if (smem > 48 * 1024)
    DMN_CUDA(cudaFuncSetAttribute(composite_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  composite_backward_kernel<<<(unsigned)((n + CB_WARPS - 1) / CB_WARPS), CB_WARPS * 32, smem, st>>>(
      raw, z, rays_d, n, s, c, keep_all, g_rgb, g_depth, g_acc, g_ins, g_weights, d_raw, accumulate);
  DMN_LAUNCH_OK();
  return 0;
}

// ================================================================================================ fp32 dW GEMMs
// The weight-gradient products the wgmma kernel does not take (gemm_tn_tc_supported): on this network only ins_linear with more
// than 64 instance logits.
constexpr int GT = 64;      // output tile GT x GT
constexpr int GK = 16;      // inner chunk

// part[split][n][k] = sum_{m in split} A[m, n] B[m, k]   (reduce_splits_kernel adds the splits into C in split order)
__global__ void __launch_bounds__(256) gemm_tn_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                                      float* __restrict__ part, int64_t M, int N, int K, int64_t rows_per_split) {
  __shared__ float As[GK][GT];
  __shared__ float Bs[GK][GT];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n0 = blockIdx.x * GT, k0 = blockIdx.y * GT;
  const int64_t mb = (int64_t)blockIdx.z * rows_per_split;
  const int64_t me = (mb + rows_per_split < M) ? mb + rows_per_split : M;
  float acc[4][4] = {};
  for (int64_t m0 = mb; m0 < me; m0 += GK) {
    for (int idx = tid; idx < GK * GT; idx += 256) {
      const int r = idx / GT, c = idx % GT;
      const int64_t m = m0 + r;
      As[r][c] = (m < me && n0 + c < N) ? A[m * lda + n0 + c] : 0.0f;
      Bs[r][c] = (m < me && k0 + c < K) ? B[m * ldb + k0 + c] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* mine = part + (size_t)blockIdx.z * N * K;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int nn = n0 + ty + 16 * i;
    if (nn >= N) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tx + 16 * j;
      if (k < K) mine[(size_t)nn * K + k] = acc[i][j];
    }
  }
}

// 128x128 register-tiled variant for operands whose widths and row strides are multiples of 4 floats (e.g. ins_num 127); the
// generic kernel above takes the other widths (e.g. ins_num 93).
constexpr int BT = 128;     // output tile BT x BT, 256 threads, 8x8 outputs per thread
constexpr int BK = 8;       // inner slice

__device__ __forceinline__ void fma_8x8(float (&acc)[8][8], const float* __restrict__ as, const float* __restrict__ bs, int ty, int tx) {
  const float4 a0 = *reinterpret_cast<const float4*>(as + ty * 8), a1 = *reinterpret_cast<const float4*>(as + ty * 8 + 4);
  const float4 b0 = *reinterpret_cast<const float4*>(bs + tx * 8), b1 = *reinterpret_cast<const float4*>(bs + tx * 8 + 4);
  const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
  const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
}

// part[split][n][k] = sum_{m in split} A[m, n] B[m, k].  N % 4 == 0, K % 4 == 0, lda/ldb % 4 == 0; rows_per_split % 8 == 0.
__global__ void __launch_bounds__(256) gemm_tn_big_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                                          float* __restrict__ part, int64_t M, int N, int K, int64_t rows_per_split) {
  __shared__ __align__(16) float As[2][BK][BT];
  __shared__ __align__(16) float Bs[2][BK][BT];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n0 = blockIdx.x * BT, k0 = blockIdx.y * BT;
  const int64_t mb = (int64_t)blockIdx.z * rows_per_split;
  const int64_t me = (mb + rows_per_split < M) ? mb + rows_per_split : M;
  const int lr = tid >> 5, lc = (tid & 31) * 4;         // slice row lr (sample), columns lc..lc+3
  float acc[8][8] = {};
  float4 ra, rb;
  auto load = [&](int64_t m0) {
    const int64_t m = m0 + lr;
    const bool ok = m < me;
    ra = (ok && n0 + lc < N) ? *reinterpret_cast<const float4*>(A + m * lda + n0 + lc) : make_float4(0.f, 0.f, 0.f, 0.f);
    rb = (ok && k0 + lc < K) ? *reinterpret_cast<const float4*>(B + m * ldb + k0 + lc) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  auto stash = [&](int buf) {
    *reinterpret_cast<float4*>(&As[buf][lr][lc]) = ra;
    *reinterpret_cast<float4*>(&Bs[buf][lr][lc]) = rb;
  };
  load(mb);
  stash(0);
  __syncthreads();
  int buf = 0;
  for (int64_t m0 = mb; m0 < me; m0 += BK) {
    if (m0 + BK < me) load(m0 + BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) fma_8x8(acc, As[buf][kk], Bs[buf][kk], ty, tx);
    if (m0 + BK < me) stash(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }
  float* mine = part + (size_t)blockIdx.z * N * K;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int nn = n0 + ty * 8 + i;
    if (nn >= N) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + tx * 8 + j;
      if (k < K) mine[(size_t)nn * K + k] = acc[i][j];
    }
  }
}

// C[n, k] += sum_split part[split][n][k], the splits added in order (reproducible bit for bit).  A block owns 32 consecutive
// entries; its 8 warps take the splits round robin and their 8 sums are added in warp order.
__global__ void __launch_bounds__(256) reduce_splits_kernel(const float* __restrict__ part, int splits, int N, int K,
                                                            float* __restrict__ Cm, int ldc) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t nk = (int64_t)N * K, e = (int64_t)blockIdx.x * 32 + lane;
  float s = 0.0f;
  if (e < nk)
    for (int z = warp; z < splits; z += 8) s += __ldcs(part + (size_t)z * nk + e);
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && e < nk) {
    float t = 0.0f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][lane];
    Cm[(size_t)(e / K) * ldc + e % K] += t;
  }
}

// Splits of the fp32 dW GEMMs: at most this many for m samples (the split heights below are at least 256 rows, the counts at
// most 4 * 132), each a [N x K] partial with N * K <= TN_PART_ENTRIES (ins_linear: up to 128 logits x 128 hidden units).
constexpr int64_t TN_MAX_SPLITS = 4 * 132;
constexpr int64_t TN_PART_ENTRIES = 128 * 128;
static int64_t tn_part_floats(int64_t m) {
  const int64_t s = (m + 255) / 256;
  return (s < TN_MAX_SPLITS ? s : TN_MAX_SPLITS) * TN_PART_ENTRIES;
}

// C[n, k] += sum_m A[m, n] B[m, k] (C zero-initialised by the caller); part: tn_part_floats(M) floats of scratch.
static int gemm_tn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int64_t M, int N, int K, float* part,
                   cudaStream_t st) {
  DMN_CHECK((int64_t)N * K <= TN_PART_ENTRIES, "mlp_backward: %d x %d weight gradient exceeds the split scratch", N, K);
  const bool aligned = ((uintptr_t)A % 16 == 0) && ((uintptr_t)B % 16 == 0);
  const bool big = aligned && N % 4 == 0 && K % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && N >= 64 && K >= 64;
  const int tile = big ? BT : GT, step = big ? BK : GK, min_rows = big ? 512 : 256;
  const int tiles = ((N + tile - 1) / tile) * ((K + tile - 1) / tile);
  int64_t splits = ((big ? 3 : 4) * 132 + tiles - 1) / tiles;
  int64_t rows = (M + splits - 1) / splits;
  rows = ((rows + step - 1) / step) * step;
  if (rows < min_rows) rows = min_rows;
  splits = (M + rows - 1) / rows;
  DMN_CHECK(splits * N * K <= tn_part_floats(M), "mlp_backward: %lld splits exceed the split scratch", (long long)splits);
  dim3 grid((unsigned)((N + tile - 1) / tile), (unsigned)((K + tile - 1) / tile), (unsigned)splits);
  if (big) gemm_tn_big_kernel<<<grid, 256, 0, st>>>(A, lda, B, ldb, part, M, N, K, rows);
  else gemm_tn_kernel<<<grid, 256, 0, st>>>(A, lda, B, ldb, part, M, N, K, rows);
  DMN_LAUNCH_OK();
  reduce_splits_kernel<<<(unsigned)(((int64_t)N * K + 31) / 32), 256, 0, st>>>(part, (int)splits, N, K, C, ldc);
  DMN_LAUNCH_OK();
  return 0;
}

// Column sums of d_out (the output-layer bias gradients) in a fixed order: pass 1 gives one partial row per block (warps over
// rows, lanes over 32 columns, the 8 warp sums added in warp order), pass 2 adds the partial rows in block order.
constexpr int COLSUM_BLOCKS = 4 * 132;
constexpr int COLSUM_MAX_C = 4 + DMNERF_MAX_INS + 1;
__global__ void __launch_bounds__(256) colsum_rows_kernel(const float* __restrict__ A, int C, int64_t m, int64_t rows_per_block,
                                                          float* __restrict__ part) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
  const int64_t r1 = (r0 + rows_per_block < m) ? r0 + rows_per_block : m;
  for (int c0 = 0; c0 < C; c0 += 32) {
    const int c = c0 + lane;
    float s = 0.0f;
    if (c < C)
      for (int64_t r = r0 + warp; r < r1; r += 8) s += __ldg(A + r * C + c);
    red[warp][lane] = s;
    __syncthreads();
    if (warp == 0 && c < C) {
      float t = 0.0f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += red[w][lane];
      part[(size_t)blockIdx.x * C + c] = t;
    }
    __syncthreads();
  }
}

__global__ void colsum_finish_kernel(const float* __restrict__ part, int C, int blocks, float* __restrict__ out) {
  const int c = threadIdx.x;
  if (c >= C) return;
  float s = 0.0f;
  for (int b = 0; b < blocks; ++b) s += part[(size_t)b * C + c];
  out[c] = s;
}

static int colsum_fixed(const float* A, int C, int64_t m, float* part, float* out, cudaStream_t st) {
  const int64_t rows = (m + COLSUM_BLOCKS - 1) / COLSUM_BLOCKS;
  const int blocks = (int)((m + rows - 1) / rows);
  colsum_rows_kernel<<<blocks, 256, 0, st>>>(A, C, m, rows, part);
  DMN_LAUNCH_OK();
  colsum_finish_kernel<<<1, COLSUM_MAX_C, 0, st>>>(part, C, blocks, out);
  DMN_LAUNCH_OK();
  return 0;
}

// [S1 | S2], dY0..dY7, [S1 | S2]^T h7, its column sums, the column sums of d_out, then the partial rows of those column sums and
// the split partials of the fp32 dW GEMMs
size_t mlp_backward_scratch_floats(int64_t m) {
  return (size_t)m * (256 + 8 * 256) + 256 * 256 + 256 + 256 + (size_t)COLSUM_BLOCKS * COLSUM_MAX_C + (size_t)tn_part_floats(m);
}

// Small dense products of the folded head gradients (128..256 x 256 outputs, contraction 128..256): 16 x 16 output tiles, one
// output per thread, so that the launch fills the machine (a 64 x 64 tiling runs these on 8-16 CTAs at ~35 us apiece).
//   small_nt_kernel:  C[m, n] = sum_k A[m, k] W[n, k] + rowscale[m] * bias[n]
//   small_tn_kernel:  C[n, k] = sum_m A[m, n] B[m, k]                          (M small: the whole contraction in one CTA)
constexpr int ST = 16;
__global__ void __launch_bounds__(ST * ST) small_nt_kernel(const float* __restrict__ A, int lda, const float* __restrict__ W, int ldw,
                                                           const float* __restrict__ rowscale, const float* __restrict__ bias,
                                                           float* __restrict__ Cm, int ldc, int M, int N, int K) {
  __shared__ float As[ST][ST + 1], Ws[ST][ST + 1];
  const int tx = threadIdx.x & (ST - 1), ty = threadIdx.x / ST;
  const int m = blockIdx.x * ST + ty, n = blockIdx.y * ST + tx;
  float acc = 0.0f;
  for (int k0 = 0; k0 < K; k0 += ST) {
    As[ty][tx] = (m < M && k0 + tx < K) ? A[(size_t)m * lda + k0 + tx] : 0.0f;                       // As[row m][k]
    const int wn = blockIdx.y * ST + ty;
    Ws[ty][tx] = (wn < N && k0 + tx < K) ? W[(size_t)wn * ldw + k0 + tx] : 0.0f;                     // Ws[row n][k]
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < ST; ++kk) acc = fmaf(As[ty][kk], Ws[tx][kk], acc);
    __syncthreads();
  }
  if (m < M && n < N) Cm[(size_t)m * ldc + n] = acc + (rowscale ? rowscale[m] * bias[n] : 0.0f);
}

__global__ void __launch_bounds__(ST * ST) small_tn_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                                           float* __restrict__ Cm, int ldc, int M, int N, int K) {
  __shared__ float As[ST][ST + 1], Bs[ST][ST + 1];
  const int tx = threadIdx.x & (ST - 1), ty = threadIdx.x / ST;
  const int n = blockIdx.x * ST + ty, k = blockIdx.y * ST + tx;
  float acc = 0.0f;
  for (int m0 = 0; m0 < M; m0 += ST) {
    As[ty][tx] = (m0 + ty < M && blockIdx.x * ST + tx < N) ? A[(size_t)(m0 + ty) * lda + blockIdx.x * ST + tx] : 0.0f;   // As[m][n]
    Bs[ty][tx] = (m0 + ty < M && k < K) ? B[(size_t)(m0 + ty) * ldb + k] : 0.0f;                                          // Bs[m][k]
    __syncthreads();
#pragma unroll
    for (int mm = 0; mm < ST; ++mm) acc = fmaf(As[mm][ty], Bs[mm][tx], acc);
    __syncthreads();
  }
  if (n < N && k < K) Cm[(size_t)n * ldc + k] = acc;
}

static int small_nt(const float* A, int lda, const float* W, int ldw, const float* rowscale, const float* bias, float* C, int ldc,
                    int M, int N, int K, cudaStream_t st) {
  small_nt_kernel<<<dim3((M + ST - 1) / ST, (N + ST - 1) / ST), ST * ST, 0, st>>>(A, lda, W, ldw, rowscale, bias, C, ldc, M, N, K);
  DMN_LAUNCH_OK();
  return 0;
}
static int small_tn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, cudaStream_t st) {
  small_tn_kernel<<<dim3((N + ST - 1) / ST, (K + ST - 1) / ST), ST * ST, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K);
  DMN_LAUNCH_OK();
  return 0;
}

// The training backward with the gradient chain (bwd_chain.cu) and the heads folded like in the forward:
//   S1 = d rgb_hid, S2 = d ins_hid                      (bwd_heads_kernel, masks from ActPlanes::bits)
//   dY7..dY0                                            (launch_bwd_chain: one masked wgmma dX GEMM per layer)
//   dW(l) = dY(l)^T X(l-1), db(l) = colsum dY(l)         (batched wgmma dW GEMMs over the saved planes)
//   P = S1^T h7, Q = S2^T h7  ->  the four feature / hidden head gradients by small dense products:
//     dW_rgb_hid[:, :256] = P W_rf^T + c1 (x) b_rf,  dW_rgb_feat = W_rh[:, :256]^T P,  db_rgb_feat = W_rh[:, :256]^T c1   (c1 = colsum S1)
//     (rgb_feat = h7 W_rf^T + b_rf is never materialised; same for the instance branch with Q, c2)
// Every sum over the samples runs in a fixed order, so the 30 gradients are reproducible bit for bit from run to run.
static int mlp_backward_chain(const NetParams& p, const UmmaWeights& packed, float* acts, const float* d_out, int64_t m,
                              float* const* grads, float* scratch, bool masks_saved, cudaStream_t st) {
  const int ins1 = p.ins_num + 1, C = 4 + ins1;
  const ActPlanes ap = act_planes(acts, m);
  float* S12 = scratch;                               // d rgb_hid | d ins_hid  [m,256]
  float* dY[8];
  for (int l = 0; l < 8; ++l) dY[l] = S12 + m * 256 + (size_t)l * m * 256;
  float* PQ = dY[7] + m * 256;                        // [S1 | S2]^T h7: rows 0..127 = P, 128..255 = Q
  float* c12 = PQ + 256 * 256;                        // column sums of S1 | S2
  float* cs = c12 + 256;                              // column sums of d_out [C]
  float* cs_part = cs + 256;                          // their partial rows [COLSUM_BLOCKS][C]
  float* tn_part = cs_part + (size_t)COLSUM_BLOCKS * COLSUM_MAX_C;        // split partials of the fp32 dW GEMM
  float* P = PQ, *Q = PQ + 128 * 256, *c1 = c12, *c2 = c12 + 128;
  auto gw = [&](int l) { return grads[2 * l]; };
  auto gb = [&](int l) { return grads[2 * l + 1]; };
  DMN_CUDA(cudaMemsetAsync(PQ, 0, (256 * 256 + 256 + 256) * sizeof(float), st));
  int rc = 0;
#define R(x) do { if ((rc = (x))) return rc; } while (0)
  // Every weight-gradient product of the network contracts over the same m samples and all their operands exist once the
  // gradient chain has run: they are queued by shape class and each class goes out as ONE batched tensor-core launch
  // (launch_gemm_tn_tc_batch) -- 3 GEMM + 3 reduction launches per network instead of 14 + 14.
  struct Queue { TnProblem p[TN_MAX_BATCH]; int n = 0, N = 0; } q_wide, q_in256, q_in128;      // [256 x 256], [256 x <=64], [128 x <=64]
  auto flush = [&](Queue& q) -> int {
    const int r = q.n ? launch_gemm_tn_tc_batch(q.p, q.n, m, q.N, st) : 0;
    q.n = 0;
    return r;
  };
  auto dW = [&](const float* A, int lda, const float* B, int ldb, float* Cw, int ldc, int N, int K, float* colsum_out = nullptr,
                int64_t b_cm = 0) -> int {
    TnProblem pr;
    Queue* q = nullptr;
    if (gemm_tn_tc_supported(N, K) && (K <= 64 || N == 256)) {
      pr.A = A; pr.lda = lda; pr.B = B; pr.ldb = ldb; pr.K = K; pr.transpose = 0; pr.colsum = colsum_out; pr.b_cm = b_cm;
      q = (K > 64) ? &q_wide : (N == 256 ? &q_in256 : &q_in128);
      q->N = N;
    } else if (!colsum_out && !b_cm && K > 64 && gemm_tn_tc_supported(K, N)) {      // narrow dY, wide X: (X^T dY)^T
      pr.A = B; pr.lda = ldb; pr.B = A; pr.ldb = lda; pr.K = N; pr.transpose = 1; pr.colsum = nullptr; pr.b_cm = 0;
      q = (K == 256) ? &q_in256 : &q_in128;
      q->N = K;
    } else {
      DMN_CHECK(!colsum_out && !b_cm, "mlp_backward: no kernel for the %d x %d weight gradient", N, K);
      return gemm_tn(A, lda, B, ldb, Cw, ldc, m, N, K, tn_part, st);
    }
    pr.ldc = ldc; pr.C = Cw;
    if (q->n == TN_MAX_BATCH) { const int r = flush(*q); if (r) return r; }
    q->p[q->n++] = pr;
    return 0;
  };
  if (!masks_saved) R(launch_mask_bits(acts, m, st));          // exact-fp32 forward: masks from its planes
  const float* d_rgb = d_out;
  const float* d_sig = d_out + 3;
  const float* d_ins = d_out + 4;
  R(launch_bwd_heads(p, d_out, m, ap.bits, S12, st));
  R(launch_bwd_chain(packed, p, S12, d_out, ap, m, dY, st));
  // ---- folded head layers (dm_nerf.py:89-99): one product against h7 for both branches; trunk (dm_nerf.py:83-87)
  R(dW(S12, 256, ap.h[7], 256, PQ, 256, 256, 256, c12));
  for (int l = 7; l >= 1; --l) R(dW(dY[l], 256, ap.h[l - 1], 256, gw(l), layer_in(l), 256, 256, gb(l)));
  R(flush(q_wide));
  // ---- input columns: layer 0 and the skip input [h, pts] of layer 5 (embedded position, column-major plane), density weights
  R(dW(dY[0], 256, ap.emb, CH_IN, gw(0), layer_in(0), 256, CH_POS, gb(0), m));
  R(dW(dY[5], 256, ap.emb, CH_IN, gw(5) + 256, layer_in(5), 256, CH_POS, nullptr, m));
  R(dW(d_sig, C, ap.h[7], 256, gw(L_DENSITY), 256, 1, 256));
  R(flush(q_in256));
  // ---- output layers (dm_nerf.py:101-103) and the view-direction columns of the colour hidden layer
  R(dW(d_rgb, C, ap.rgb_hid, 128, gw(L_RGB_OUT), 128, 3, 128));
  R(dW(d_ins, C, ap.ins_hid, 128, gw(L_INS_OUT), 128, ins1, 128));
  R(dW(S12, 256, ap.emb + (int64_t)CH_POS * m, CH_IN, gw(L_RGB_HID) + 256, 283, 128, CH_DIR, nullptr, m));
  R(flush(q_in128));
  // the three output bias gradients from one sweep over d_out
  R(colsum_fixed(d_out, C, m, cs_part, cs, st));
  DMN_CUDA(cudaMemcpyAsync(gb(L_RGB_OUT), cs, 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  DMN_CUDA(cudaMemcpyAsync(gb(L_DENSITY), cs + 3, sizeof(float), cudaMemcpyDeviceToDevice, st));
  DMN_CUDA(cudaMemcpyAsync(gb(L_INS_OUT), cs + 4, ins1 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  // ---- folded head layers, small products on P / Q
  R(small_nt(P, 256, p.w[L_RGB_FEAT], 256, c1, p.b[L_RGB_FEAT], gw(L_RGB_HID), 283, 128, 256, 256, st));
  R(small_nt(Q, 256, p.w[L_INS_FEAT], 256, c2, p.b[L_INS_FEAT], gw(L_INS_HID), 256, 128, 256, 256, st));
  DMN_CUDA(cudaMemcpyAsync(gb(L_RGB_HID), c1, 128 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  DMN_CUDA(cudaMemcpyAsync(gb(L_INS_HID), c2, 128 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  R(small_tn(p.w[L_RGB_HID], 283, P, 256, gw(L_RGB_FEAT), 256, 128, 256, 256, st));                // W_rh[:, :256]^T P
  R(small_tn(p.w[L_RGB_HID], 283, c1, 1, gb(L_RGB_FEAT), 1, 128, 256, 1, st));
  R(small_tn(p.w[L_INS_HID], 256, Q, 256, gw(L_INS_FEAT), 256, 128, 256, 256, st));
  R(small_tn(p.w[L_INS_HID], 256, c2, 1, gb(L_INS_FEAT), 1, 128, 256, 1, st));
#undef R
  return 0;
}

// grads: 30 device pointers in state_dict order (weight, bias per layer); overwritten with the gradient of this call.
int launch_mlp_backward(const NetParams& p, const UmmaWeights& packed, float* acts, const float* d_out, int64_t m, float* const* grads,
                        float* scratch, int flags, cudaStream_t st) {
  DMN_CHECK(p.bound, "mlp_backward: weights not bound");
  DMN_CHECK(umma_available(packed), "mlp_backward: weights not packed (call dmnerf_set_weights first)");
  const bool prezeroed = (flags & 2) != 0;      // flags: bit 0 = the forward wrote the ReLU bit planes, bit 1 = grads already zero
  for (int l = 0; l < N_LAYERS; ++l) {
    DMN_CHECK(grads[2 * l] && grads[2 * l + 1], "mlp_backward: gradient buffer %d is NULL", 2 * l);
    if (prezeroed) continue;
    DMN_CUDA(cudaMemsetAsync(grads[2 * l], 0, (size_t)layer_out(l, p.ins_num) * layer_in(l) * sizeof(float), st));
    DMN_CUDA(cudaMemsetAsync(grads[2 * l + 1], 0, (size_t)layer_out(l, p.ins_num) * sizeof(float), st));
  }
  if (m == 0) return 0;
  return mlp_backward_chain(p, packed, acts, d_out, m, grads, scratch, (flags & 1) != 0, st);
}

}  // namespace dmnerf
