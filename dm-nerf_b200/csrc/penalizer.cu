// "Emptiness" regulariser on the per-sample object logits (networks/penalizer.py:5-62, called by train_dmsr.py:53-60) and its
// gradient: the one training-time consumer of the per-sample network outputs raw[N,S,C].
//
//   L = sum_{before} air * BCE_k(sigmoid(raw_k), [k == last]) / (K * max(#before, 1e-8))          (penalizer.py:36-43)
//     + sum_{middle} g * -log(1 - sigmoid(raw_last) + 1e-8)   /      max(#middle, 1e-8)           (penalizer.py:46-52)
//   g = exp(-d^2 / (2 w^2)) / (0.4 sqrt(2 pi)) + 1e-8,  air = 1 - g,  d = (depth - z) |ray_d|      (penalizer.py:7-24)
//   before: z |d| < (depth - tol) |d|;  after: z |d| > (depth + tol) |d|;  middle = 1 - (before + after)   (penalizer.py:27-29)
//
// Two launches, both HBM-streaming with the rows of raw staged through shared memory (coalesced):
//   penalizer_partial_kernel the two mask populations (integers: exact), the two masked sums (fp64 accumulation of fp32
//                            terms, in an order fixed by the sizes) and the finalisation by the last block, in one pass over raw
//   penalizer_grad_kernel    d L / d raw * upstream gradient (a device scalar: no host synchronisation); writes every channel
//                            (zeros for rgb / sigma), so the caller needs no zero-fill
// Not folded into the composite kernel: the masks need the finished depth map of the ray (a second sweep over its samples either
// way), the tolerance / width arguments only arrive with the separate reference call (train_dmsr.py:53-60), and raw[N,S,C] has to
// exist in HBM for the composite backward in any case -- the fold would save one 14 MB read per network.
#include <cstdint>

#include "common.cuh"
#include "ray_ops.cuh"

namespace dmnerf {

struct PenState {               // scratch of one call (device): masks' populations, partial sums, block counter
  unsigned long long n_before, n_middle;
  double sum_before, sum_middle;
  unsigned int blocks_done, pad;
};

__device__ __forceinline__ void pen_geometry(const float* __restrict__ z, const float* __restrict__ depth, const float* __restrict__ rays_d,
                                             int64_t idx, int s, float tol, float w, float& g, bool& before, bool& middle) {
  const int64_t ray = idx / s;
  const float d0 = rays_d[ray * 3], d1 = rays_d[ray * 3 + 1], d2 = rays_d[ray * 3 + 2];
  const float norm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2)));   // penalizer.py:13
  const float dep = depth[ray];
  const float front = __fmul_rn(__fsub_rn(dep, tol), norm), back = __fmul_rn(__fadd_rn(dep, tol), norm);     // :14-17
  const float pos = __fmul_rn(z[idx], norm), surf = __fmul_rn(dep, norm);                                    // :18-19
  const float dd = __fsub_rn(surf, pos);                                                                     // :22
  const float two_w2 = __fmul_rn(2.0f, __fmul_rn(w, w));
  const float denom = __fmul_rn(0.4f, sqrtf(6.283185307179586f));                                            // deta_h sqrt(2 pi)
  g = __fadd_rn(__fdiv_rn(expf(__fdiv_rn(-__fmul_rn(dd, dd), two_w2)), denom), 1e-8f);                       // :7-8
  before = pos < front;                                                                                      // :27
  const bool after = pos > back;                                                                             // :28
  middle = !(before || after);                                                                               // :29
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
  return v;
}

// Samples per block: the block's rows of raw ([tile, C] contiguous floats) are staged through shared memory so that the global
// traffic is fully coalesced (a thread-per-sample walk over rows of 18..132 floats touches partial sectors only).
static int pen_tile(int c) { return c <= 48 ? 256 : (c <= 96 ? 128 : 64); }

// The tile's rows take exactly 48 KB at the widest C of a tile size (48, 96); with the forward's static shared memory that is
// over the default per-block limit, so a launch opts in to the tile's size whenever it reaches it.
static int pen_smem(const void* kernel, size_t smem) {
  if (smem >= 40 * 1024) DMN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return 0;
}

// This block's two masked sums (fp64 accumulation of fp32 terms) and two mask populations, valid in thread 0; the block's
// rows of raw are staged through shared memory.
__device__ __forceinline__ void pen_block_terms(const float* __restrict__ raw, const float* __restrict__ z, const float* __restrict__ depth,
                                                const float* __restrict__ rays_d, int64_t total, int s, int c, float tol, float w,
                                                double& tb, double& tm, unsigned long long& cb, unsigned long long& cm) {
  extern __shared__ float sraw[];
  const int tile = blockDim.x;
  const int64_t idx0 = (int64_t)blockIdx.x * tile;
  const int n_here = (int)((total - idx0 < tile) ? total - idx0 : tile);
  for (int i = threadIdx.x; i < n_here * c; i += tile) sraw[i] = raw[idx0 * c + i];
  __syncthreads();
  const int64_t idx = idx0 + threadIdx.x;
  const int K = c - 4;
  double sb = 0.0, sm = 0.0;
  bool before = false, middle = false;
  if ((int)threadIdx.x < n_here) {
    float g;
    pen_geometry(z, depth, rays_d, idx, s, tol, w, g, before, middle);
    const float* r = sraw + threadIdx.x * c + 4;
    if (before) {
      const float air = __fsub_rn(1.0f, g);                                                                  // :24
      float acc = 0.0f;
      for (int k = 0; k < K; ++k) {
        const float p = sigmoidf_acc(r[k]);                                                                  // :33
        const float term = (k == K - 1) ? -logf(__fadd_rn(p, 1e-8f)) : -logf(__fadd_rn(__fsub_rn(1.0f, p), 1e-8f));   // :39
        acc = __fadd_rn(acc, __fmul_rn(term, air));                                                          // :40-41
      }
      sb = (double)acc;
    }
    if (middle) {
      const float p = sigmoidf_acc(r[K - 1]);
      sm = (double)__fmul_rn(-logf(__fadd_rn(__fsub_rn(1.0f, p), 1e-8f)), g);                                // :49-51
    }
  }
  const unsigned nb = __popc(__ballot_sync(FULL, before)), nm = __popc(__ballot_sync(FULL, middle));
  sb = warp_sum_d(sb);
  sm = warp_sum_d(sm);
  __shared__ double sh_b[8], sh_m[8];
  __shared__ unsigned sh_nb[8], sh_nm[8];
  const int wid = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { sh_b[wid] = sb; sh_m[wid] = sm; sh_nb[wid] = nb; sh_nm[wid] = nm; }
  __syncthreads();
  tb = 0.0; tm = 0.0; cb = 0; cm = 0;
  if (threadIdx.x == 0)
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { tb += sh_b[i]; tm += sh_m[i]; cb += sh_nb[i]; cm += sh_nm[i]; }
}

// penalizer.py:42-43, 52-53
__device__ __forceinline__ float pen_finalise(unsigned long long n_before, unsigned long long n_middle, double sum_before,
                                              double sum_middle, int K) {
  const double nbt = fmax((double)n_before, 1e-8), nmt = fmax((double)n_middle, 1e-8);
  return (float)(sum_before / ((double)K * nbt) + sum_middle / nmt);
}

// Forward in ONE pass over the batch or over one shard of it: the populations and masked sums, summed in an order fixed by the
// size alone (no floating-point atomics).  Every block writes its terms to its own slot after the PenState head, and the last
// block to finish adds the slots with a fixed-shape reduction into the head and writes the loss of those sums.  A single
// process reads that loss; the shards of a batch gather their heads and merge them (penalizer_merge_kernel), which at one
// shard gives the same head and loss bit for bit.
struct PenBlock {
  double sb, sm;
  unsigned long long nb, nm;
};

__global__ void penalizer_partial_kernel(const float* __restrict__ raw, const float* __restrict__ z, const float* __restrict__ depth,
                                         const float* __restrict__ rays_d, int64_t total, int s, int c, float tol, float w,
                                         PenState* st, PenBlock* blocks, float* __restrict__ loss) {
  double tb, tm;
  unsigned long long cb, cm;
  pen_block_terms(raw, z, depth, rays_d, total, s, c, tol, w, tb, tm, cb, cm);
  __shared__ bool last;
  if (threadIdx.x == 0) {
    blocks[blockIdx.x] = PenBlock{tb, tm, cb, cm};
    __threadfence();
    last = atomicAdd(&st->blocks_done, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double sb = 0.0, sm = 0.0;
  unsigned long long nb = 0, nm = 0;
#pragma unroll 4
  for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x) {
    sb += __ldcg(&blocks[b].sb); sm += __ldcg(&blocks[b].sm); nb += __ldcg(&blocks[b].nb); nm += __ldcg(&blocks[b].nm);
  }
  sb = warp_sum_d(sb);
  sm = warp_sum_d(sm);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { nb += __shfl_xor_sync(FULL, nb, d); nm += __shfl_xor_sync(FULL, nm, d); }
  __shared__ PenBlock wsum[8];
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = PenBlock{sb, sm, nb, nm};
  __syncthreads();
  if (threadIdx.x == 0) {
    PenBlock t{0.0, 0.0, 0, 0};
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { t.sb += wsum[i].sb; t.sm += wsum[i].sm; t.nb += wsum[i].nb; t.nm += wsum[i].nm; }
    st->sum_before = t.sb; st->sum_middle = t.sm; st->n_before = t.nb; st->n_middle = t.nm;
    loss[0] = pen_finalise(t.nb, t.nm, t.sb, t.sm, c - 4);
  }
}

// `world` shard heads added in shard order into `out` (what penalizer_grad_kernel reads) and the loss of the whole batch.
__global__ void penalizer_merge_kernel(const PenState* __restrict__ parts, int world, int K, PenState* __restrict__ out,
                                       float* __restrict__ loss) {
  PenState t{};
  for (int r = 0; r < world; ++r) {
    t.n_before += parts[r].n_before; t.n_middle += parts[r].n_middle;
    t.sum_before += parts[r].sum_before; t.sum_middle += parts[r].sum_middle;
  }
  *out = t;
  loss[0] = pen_finalise(t.n_before, t.n_middle, t.sum_before, t.sum_middle, K);
}

// d_raw = g_loss * dL/d raw: every channel of every row is written (channels 0..3 get zeros), through shared memory, so the
// caller needs no zero-fill.  accumulate != 0: d_raw[..., 4:] += the gradient (direct strided path, channels 0..3 untouched).
__global__ void penalizer_grad_kernel(const float* __restrict__ raw, const float* __restrict__ z, const float* __restrict__ depth,
                                      const float* __restrict__ rays_d, int64_t total, int s, int c, float tol, float w,
                                      const PenState* __restrict__ st, const float* __restrict__ g_loss, float* __restrict__ d_raw,
                                      int accumulate) {
  extern __shared__ float sraw[];
  const int tile = blockDim.x;
  const int64_t idx0 = (int64_t)blockIdx.x * tile;
  const int n_here = (int)((total - idx0 < tile) ? total - idx0 : tile);
  for (int i = threadIdx.x; i < n_here * c; i += tile) sraw[i] = raw[idx0 * c + i];
  __syncthreads();
  const int K = c - 4;
  if ((int)threadIdx.x < n_here) {
    const int64_t idx = idx0 + threadIdx.x;
    float g;
    bool before, middle;
    pen_geometry(z, depth, rays_d, idx, s, tol, w, g, before, middle);
    const float up = g_loss[0];
    const float cb = up * (float)(1.0 / ((double)K * fmax((double)st->n_before, 1e-8)));
    const float cm = up * (float)(1.0 / fmax((double)st->n_middle, 1e-8));
    const float air = 1.0f - g;
    float* r = sraw + threadIdx.x * c;
    r[0] = 0.0f; r[1] = 0.0f; r[2] = 0.0f; r[3] = 0.0f;
    for (int k = 0; k < K; ++k) {
      float gr = 0.0f;
      if (before || (middle && k == K - 1)) {
        const float p = sigmoidf_acc(r[4 + k]);
        const float dp = p * (1.0f - p);                                   // d sigmoid
        // d/dx -log(1 - p + eps) = dp / (1 - p + eps);   d/dx -log(p + eps) = -dp / (p + eps)
        if (before) gr += cb * air * ((k == K - 1) ? -dp / (p + 1e-8f) : dp / (1.0f - p + 1e-8f));
        if (middle && k == K - 1) gr += cm * g * dp / (1.0f - p + 1e-8f);
      }
      r[4 + k] = gr;
    }
  }
  __syncthreads();
  if (!accumulate) {
    for (int i = threadIdx.x; i < n_here * c; i += tile) d_raw[idx0 * c + i] = sraw[i];
  } else {
    for (int i = threadIdx.x; i < n_here * c; i += tile)
      if (i % c >= 4) d_raw[idx0 * c + i] += sraw[i];
  }
}

int launch_penalizer_backward(const float* raw, const float* z, const float* depth, const float* rays_d, int64_t n, int s, int c,
                              float tol, float w, const void* state, const float* g_loss, float* d_raw, int accumulate,
                              cudaStream_t st) {
  DMN_CHECK(c > 4 && c <= 4 + DMNERF_MAX_INS + 1 && s >= 1, "penalizer: bad sizes s=%d c=%d", s, c);
  const int64_t total = n * s;
  if (total == 0) return 0;
  const int tile = pen_tile(c);
  const unsigned grid = (unsigned)((total + tile - 1) / tile);
  if (pen_smem((const void*)penalizer_grad_kernel, (size_t)tile * c * sizeof(float))) return 1;
  penalizer_grad_kernel<<<grid, tile, (size_t)tile * c * sizeof(float), st>>>(raw, z, depth, rays_d, total, s, c, tol, w,
                                                                              reinterpret_cast<const PenState*>(state), g_loss, d_raw,
                                                                              accumulate);
  DMN_LAUNCH_OK();
  return 0;
}

size_t penalizer_state_bytes() { return sizeof(PenState); }

static_assert(sizeof(PenState) % alignof(PenBlock) == 0, "block slots follow the head");
size_t penalizer_partials_bytes(int64_t n, int s, int c) {
  const int64_t total = n * s;
  const int tile = pen_tile(c);
  return sizeof(PenState) + (size_t)((total + tile - 1) / tile) * sizeof(PenBlock);
}

int launch_penalizer_forward(const float* raw, const float* z, const float* depth, const float* rays_d, int64_t n, int s, int c,
                             float tol, float w, void* partials, float* loss, cudaStream_t st) {
  DMN_CHECK(c > 4 && c <= 4 + DMNERF_MAX_INS + 1 && s >= 1, "penalizer: bad sizes s=%d c=%d", s, c);
  PenState* ps = reinterpret_cast<PenState*>(partials);
  DMN_CUDA(cudaMemsetAsync(ps, 0, sizeof(PenState), st));
  const int64_t total = n * s;
  if (total == 0) {
    DMN_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), st));
    return 0;
  }
  const int tile = pen_tile(c);
  const unsigned grid = (unsigned)((total + tile - 1) / tile);
  if (pen_smem((const void*)penalizer_partial_kernel, (size_t)tile * c * sizeof(float))) return 1;
  penalizer_partial_kernel<<<grid, tile, (size_t)tile * c * sizeof(float), st>>>(raw, z, depth, rays_d, total, s, c, tol, w, ps,
                                                                                 reinterpret_cast<PenBlock*>(ps + 1), loss);
  DMN_LAUNCH_OK();
  return 0;
}

int launch_penalizer_merge(const void* states, int world, int c, void* state, float* loss, cudaStream_t st) {
  DMN_CHECK(c > 4 && c <= 4 + DMNERF_MAX_INS + 1 && world >= 1, "penalizer_merge: bad sizes world=%d c=%d", world, c);
  penalizer_merge_kernel<<<1, 1, 0, st>>>(reinterpret_cast<const PenState*>(states), world, c - 4, reinterpret_cast<PenState*>(state),
                                          loss);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
