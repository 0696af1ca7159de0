// Hungarian-matched instance loss of the training step (networks/evaluator.py:19-74, called twice per iteration by
// train_dmsr.py:38-45): the two [ins x ins] cost matrices from ONE pass over the N rays of the batch, and the gradient of the
// matched loss.  The assignment itself (scipy linear_sum_assignment on the [valid x ins] matrix, evaluator.py:45-47) either stays
// on the host like in the reference (dmnerf_hungarian_costs + scipy: one device->host hop per call) or runs on the device
// (label_rows_kernel + hungarian_assign_kernel: the same shortest-augmenting-path algorithm with the same tie rule, no hop at
// all -- the training iteration stays asynchronous end to end).
//
// gt is one-hot (evaluator.py:21-25: column v of gt_ins marks the rays whose label is the v-th smallest label present), so the
// dense [ins x ins x N] broadcast of the reference collapses to per-row sums.  With row(n) = index of ray n's label:
//   A[p]    = sum_n          log(1 - pred[n,p] + 1e-8)
//   B[g,p]  = sum_{row(n)=g} log(pred[n,p] + 1e-8)       C[g,p] = sum_{row(n)=g} log(1 - pred[n,p] + 1e-8)
//   TP[g,p] = sum_{row(n)=g} pred[n,p]                   S[p]   = sum_n pred[n,p]           cnt[g] = #{n : row(n) = g}
//   cost_ce[g,p]   = -(B[g,p] + A[p] - C[g,p]) / N                                           (evaluator.py:60)
//   cost_siou[g,p] = 1 - TP / (TP + (S[p] - TP) + (cnt[g] - TP) + 1e-6)                      (evaluator.py:63-67)
// fp32 terms, fp64 accumulation (the reference sums fp32 terms pairwise: both are ~1e-7 from the exact sum).
#include <cstdint>

#include "common.cuh"
#include "ray_ops.cuh"

namespace dmnerf {

constexpr int EV_MAX_K = DMNERF_MAX_INS + 1;

// cost_ce / cost_siou / tp of cell (g, p), and col_sum / row_count, from the fp64 sums of the batch of n rays.
__device__ __forceinline__ void write_costs(int g, int p, int k, int64_t n, double A, double S, double B, double C, double TP,
                                            double cnt, float* __restrict__ cost_ce, float* __restrict__ cost_siou,
                                            float* __restrict__ tp_out, float* __restrict__ cnt_out) {
  cost_ce[(size_t)g * k + p] = (float)(-(B + A - C) / (double)n);
  // the reference evaluates TP, FP = sum(pred) - TP, FN = sum(gt) - TP in fp32 and then TP / (TP + FP + FN + 1e-6)
  const float tpf = (float)TP, fp = __fsub_rn((float)S, tpf), fn = __fsub_rn((float)cnt, tpf);
  const float den = __fadd_rn(__fadd_rn(__fadd_rn(tpf, fp), fn), 1e-6f);
  cost_siou[(size_t)g * k + p] = __fsub_rn(1.0f, __fdiv_rn(tpf, den));
  tp_out[(size_t)g * k + p] = tpf;
  if (p == 0) cnt_out[g] = (float)cnt;
}

// The sums above, in fp64, for the batch or for one contiguous shard of it, summed in an order fixed by the size alone (no
// floating-point atomics).  One block per column p; every warp walks 32-row chunks, adds the rows of one label in lane order
// and keeps its own per-label sums; the warps' sums are added in warp order at the end.  Then either
//   FINAL = false: the shard's partials = A[k] | S[k] | B[k x k] | C[k x k] | TP[k x k] | cnt[k] (row g, column p at g * k + p),
//                  merged by hungarian_costs_merged_kernel, or
//   FINAL = true:  the costs of the whole batch (n rays) straight from these sums -- the one-shard case of the merge, and bit
//                  for bit its result, since the merge adds each partial to 0.0.
constexpr int HP_WARPS = 8;
template <bool FINAL>
__global__ void __launch_bounds__(HP_WARPS * 32) hungarian_partials_kernel(const float* __restrict__ pred,
                                                                             const int32_t* __restrict__ gt_row, int64_t n, int k,
                                                                             double* __restrict__ out, float* __restrict__ cost_ce,
                                                                             float* __restrict__ cost_siou, float* __restrict__ tp_out,
                                                                             float* __restrict__ s_out, float* __restrict__ cnt_out) {
  __shared__ double wB[HP_WARPS][EV_MAX_K], wC[HP_WARPS][EV_MAX_K], wTP[HP_WARPS][EV_MAX_K];
  __shared__ unsigned int wCnt[HP_WARPS][EV_MAX_K];
  __shared__ double stage[HP_WARPS][3][32];
  __shared__ double wA[HP_WARPS], wS[HP_WARPS];
  const int p = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int g = lane; g < k; g += 32) { wB[warp][g] = 0.0; wC[warp][g] = 0.0; wTP[warp][g] = 0.0; wCnt[warp][g] = 0u; }
  __syncwarp();
  double a = 0.0, s = 0.0;
  for (int64_t base = (int64_t)warp * 32; base < n; base += HP_WARPS * 32) {      // warp-uniform trip count
    const int64_t i = base + lane;
    int g = -1;
    double lb = 0.0, lc = 0.0, v = 0.0;
    if (i < n) {
      const float vf = pred[i * k + p];
      const float l1 = logf(__fadd_rn(__fsub_rn(1.0f, vf), 1e-8f));
      a += (double)l1;
      s += (double)vf;
      g = gt_row[i];
      if (g >= 0 && g < k) { lb = (double)logf(__fadd_rn(vf, 1e-8f)); lc = (double)l1; v = (double)vf; }
      else g = -1;
    }
    stage[warp][0][lane] = lb; stage[warp][1][lane] = lc; stage[warp][2][lane] = v;
    const unsigned grp = __match_any_sync(FULL, g);
    __syncwarp();
    if (g >= 0 && lane == __ffs(grp) - 1) {                 // the lowest lane of each label adds that label's rows in lane order
      double b = 0.0, c = 0.0, t = 0.0;
      for (unsigned m = grp; m; m &= m - 1) {
        const int j = __ffs(m) - 1;
        b += stage[warp][0][j]; c += stage[warp][1][j]; t += stage[warp][2][j];
      }
      wB[warp][g] += b; wC[warp][g] += c; wTP[warp][g] += t; wCnt[warp][g] += __popc(grp);
    }
    __syncwarp();
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { a += __shfl_xor_sync(FULL, a, d); s += __shfl_xor_sync(FULL, s, d); }
  if (lane == 0) { wA[warp] = a; wS[warp] = s; }
  __syncthreads();
  const size_t kk = (size_t)k * k;
  double* A = out; double* S = out + k; double* B = out + 2 * k; double* C = B + kk; double* TP = C + kk; double* cnt = TP + kk;
  double ta = 0.0, ts = 0.0;
  if constexpr (FINAL)                                       // every cell of the column needs A[p] and S[p]
    for (int w = 0; w < HP_WARPS; ++w) { ta += wA[w]; ts += wS[w]; }
  for (int g = threadIdx.x; g < k; g += blockDim.x) {
    double b = 0.0, c = 0.0, t = 0.0;
    unsigned int m = 0u;
    for (int w = 0; w < HP_WARPS; ++w) { b += wB[w][g]; c += wC[w][g]; t += wTP[w][g]; m += wCnt[w][g]; }
    if constexpr (FINAL) {
      write_costs(g, p, k, n, ta, ts, b, c, t, (double)m, cost_ce, cost_siou, tp_out, cnt_out);
    } else {
      B[(size_t)g * k + p] = b; C[(size_t)g * k + p] = c; TP[(size_t)g * k + p] = t;
      if (p == 0) cnt[g] = (double)m;
    }
  }
  if (threadIdx.x == 0) {
    if constexpr (FINAL) {
      s_out[p] = (float)ts;
    } else {
      for (int w = 0; w < HP_WARPS; ++w) { ta += wA[w]; ts += wS[w]; }
      A[p] = ta; S[p] = ts;
    }
  }
}

// The partials of `world` shards added in shard order, then the costs of the batch of n rays (write_costs).
__global__ void hungarian_costs_merged_kernel(const double* __restrict__ partials, int world, int64_t n, int k,
                                              float* __restrict__ cost_ce, float* __restrict__ cost_siou, float* __restrict__ tp_out,
                                              float* __restrict__ s_out, float* __restrict__ cnt_out) {
  const int p = blockIdx.x;
  const size_t kk = (size_t)k * k, stride = 3 * (size_t)k + 3 * kk;
  double A = 0.0, S = 0.0;
  for (int w = 0; w < world; ++w) { A += partials[w * stride + p]; S += partials[w * stride + k + p]; }
  for (int g = threadIdx.x; g < k; g += blockDim.x) {
    const size_t cell = 2 * (size_t)k + (size_t)g * k + p;
    double B = 0.0, C = 0.0, TP = 0.0, cnt = 0.0;
    for (int w = 0; w < world; ++w) {
      const double* q = partials + w * stride;
      B += q[cell]; C += q[cell + kk]; TP += q[cell + 2 * kk]; cnt += q[2 * k + 3 * kk + g];
    }
    write_costs(g, p, k, n, A, S, B, C, TP, cnt, cost_ce, cost_siou, tp_out, cnt_out);
  }
  if (threadIdx.x == 0) s_out[p] = (float)S;
}

// d loss / d pred for  loss = g_ce * valid_ce + g_inv * invalid_ce + g_siou * valid_siou  (evaluator.py:27-36):
//   valid_ce = mean_{g < V} cost_ce[g, col(g)],  valid_siou likewise,  invalid_ce = mean(pred[:, unmatched columns]).
// row_of_col[p] = matched gt row of prediction column p, or -1 (unmatched).  g3 = the three upstream gradients (device).
// n rows of pred are written; n_norm is the ray count of the whole batch (n_norm > n for one shard of it).  n_valid_dev = the
// number of distinct labels (device).
__global__ void ins_loss_grad_kernel(const float* __restrict__ pred, const int32_t* __restrict__ gt_row, int64_t n, int64_t n_norm,
                                     int k, const int32_t* __restrict__ row_of_col, const int32_t* __restrict__ n_valid_dev,
                                     const float* __restrict__ tp, const float* __restrict__ s_sum, const float* __restrict__ cnt,
                                     const float* __restrict__ g3, float* __restrict__ d_pred) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * k) return;
  const int n_valid = *n_valid_dev;
  if (n_valid < 1) { d_pred[idx] = 0.0f; return; }          // rejected labels: NaN loss, zero gradient, error on the next call
  const int64_t i = idx / k;
  const int p = (int)(idx % k);
  const int g = row_of_col[p];
  const float v = pred[idx];
  float d;
  if (g >= 0) {
    const bool on = gt_row[i] == g;
    const float inv_v = 1.0f / (float)n_valid;
    const float dce = on ? -1.0f / (v + 1e-8f) : 1.0f / ((1.0f - v) + 1e-8f);
    const float t = tp[(size_t)g * k + p];
    const float den = (s_sum[p] + cnt[g] - t) + 1e-6f;
    const float dsi = on ? -1.0f / den : t / (den * den);      // -(gt D - TP (1 - gt)) / D^2
    d = g3[0] * inv_v * dce / (float)n_norm + g3[2] * inv_v * dsi;
  } else {
    d = g3[1] / ((float)n_norm * (float)(k - n_valid));
  }
  d_pred[idx] = d;
}

// ---------------------------------------------------------------------------------------------------- device-side assignment
// Row of every ray = rank of its label among the distinct labels of the batch (ascending: torch.unique order, evaluator.py:21-25),
// from a presence bitmap over label values [0, 65536); n_valid = number of distinct labels.  Labels outside that range or more
// distinct labels than prediction channels: n_valid = -1 (the loss comes out NaN, its gradient zero) and the code goes to the
// status word (mapped host memory: the next ins_criterion call raises without any synchronisation).
constexpr int LBL_WORDS = 2048;            // 65536 label values
static_assert(DMNERF_LABEL_WORDS == LBL_WORDS + 1, "bitmap layout of dmnerf_ins_label_bitmap");

// Bitmap of the labels[0..n) into shared memory (1024 threads); bad_s = 1 when a label is outside [0, 65536).
__device__ __forceinline__ void label_presence(const int32_t* __restrict__ labels, int64_t n, uint32_t* bitmap, int* bad_s) {
  for (int64_t i = threadIdx.x; i < n; i += 1024) {
    const int l = labels[i];
    if (l < 0 || l >= LBL_WORDS * 32) *bad_s = 1;
    else atomicOr(&bitmap[l >> 5], 1u << (l & 31));
  }
}

// prefix[w] = number of labels present in words 0..w-1 of the bitmap (1024 threads); returns the number of labels present.
__device__ __forceinline__ int label_prefix(const uint32_t* bitmap, uint32_t* prefix, uint32_t* warp_tot) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint32_t c0 = __popc(bitmap[2 * t]), c1 = __popc(bitmap[2 * t + 1]);
  uint32_t incl = c0 + c1;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(FULL, incl, d); if (lane >= d) incl += o; }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = warp_tot[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(FULL, w, d); if (lane >= d) w += o; }
    warp_tot[lane] = w;                                      // inclusive totals of the warps
  }
  __syncthreads();
  const uint32_t excl = incl - (c0 + c1) + (warp ? warp_tot[warp - 1] : 0u);
  prefix[2 * t] = excl; prefix[2 * t + 1] = excl + c0;
  __syncthreads();
  return (int)warp_tot[31];
}

// gt_row[i] = rank of labels[i] among the labels of the bitmap (-1 for all rows when `bad`), n_valid_out, error code.
__device__ __forceinline__ void label_rank_rows(const int32_t* __restrict__ labels, int64_t n, const uint32_t* bitmap,
                                                const uint32_t* prefix, int n_valid, bool bad, int code, int32_t* __restrict__ gt_row,
                                                int32_t* __restrict__ n_valid_out, int32_t* status) {
  for (int64_t i = threadIdx.x; i < n; i += 1024) {
    const int l = labels[i];
    int row = -1;
    if (!bad && l >= 0 && l < LBL_WORDS * 32) row = (int)(prefix[l >> 5] + __popc(bitmap[l >> 5] & ((1u << (l & 31)) - 1u)));
    gt_row[i] = row;
  }
  if (threadIdx.x == 0) {
    *n_valid_out = bad ? -1 : n_valid;
    if (bad && status) atomicCAS(status, 0, code);
  }
}

__global__ void __launch_bounds__(1024) label_rows_kernel(const int32_t* __restrict__ labels, int64_t n, int k,
                                                          int32_t* __restrict__ gt_row, int32_t* __restrict__ n_valid_out,
                                                          int32_t* status) {
  __shared__ uint32_t bitmap[LBL_WORDS], prefix[LBL_WORDS];
  __shared__ uint32_t warp_tot[32];
  __shared__ int bad_s;
  const int t = threadIdx.x;
  bitmap[2 * t] = 0u; bitmap[2 * t + 1] = 0u;
  if (t == 0) bad_s = 0;
  __syncthreads();
  label_presence(labels, n, bitmap, &bad_s);
  __syncthreads();
  const int n_valid = label_prefix(bitmap, prefix, warp_tot);
  const bool bad = bad_s != 0 || n_valid > k || n_valid < 1;
  label_rank_rows(labels, n, bitmap, prefix, n_valid, bad, bad_s ? 701 : 702, gt_row, n_valid_out, status);
}

// One shard's presence bitmap: words 0..2047 over label values [0, 65536), word 2048 = 1 when a label is out of range (which
// also goes to the status word: 701).  OR is order-free, so the bitmap does not depend on scheduling.
__global__ void __launch_bounds__(1024) label_bitmap_kernel(const int32_t* __restrict__ labels, int64_t n, uint32_t* __restrict__ out,
                                                            int32_t* status) {
  __shared__ uint32_t bitmap[LBL_WORDS];
  __shared__ int bad_s;
  const int t = threadIdx.x;
  bitmap[2 * t] = 0u; bitmap[2 * t + 1] = 0u;
  if (t == 0) bad_s = 0;
  __syncthreads();
  label_presence(labels, n, bitmap, &bad_s);
  __syncthreads();
  out[2 * t] = bitmap[2 * t]; out[2 * t + 1] = bitmap[2 * t + 1];
  if (t == 0) {
    out[LBL_WORDS] = bad_s ? 1u : 0u;
    if (bad_s && status) atomicCAS(status, 0, 701);
  }
}

// label_rows_kernel on the OR of `world` shard bitmaps (rank order) for the shard's own labels: every shard ranks its rows among
// the distinct labels of the whole batch and every shard gets the same n_valid (or -1 and the same error code).
__global__ void __launch_bounds__(1024) label_rows_merged_kernel(const uint32_t* __restrict__ bitmaps, int world,
                                                                 const int32_t* __restrict__ labels, int64_t n, int k,
                                                                 int32_t* __restrict__ gt_row, int32_t* __restrict__ n_valid_out,
                                                                 int32_t* status) {
  __shared__ uint32_t bitmap[LBL_WORDS], prefix[LBL_WORDS];
  __shared__ uint32_t warp_tot[32];
  __shared__ int bad_s;
  const int t = threadIdx.x;
  uint32_t b0 = 0u, b1 = 0u, flag = 0u;
  for (int w = 0; w < world; ++w) {
    const uint32_t* q = bitmaps + (size_t)w * (LBL_WORDS + 1);
    b0 |= q[2 * t]; b1 |= q[2 * t + 1]; flag |= q[LBL_WORDS];
  }
  bitmap[2 * t] = b0; bitmap[2 * t + 1] = b1;
  if (t == 0) bad_s = flag != 0u;
  __syncthreads();
  const int n_valid = label_prefix(bitmap, prefix, warp_tot);
  const bool bad = bad_s != 0 || n_valid > k || n_valid < 1;
  label_rank_rows(labels, n, bitmap, prefix, n_valid, bad, bad_s ? 701 : 702, gt_row, n_valid_out, status);
}

// scipy.optimize.linear_sum_assignment (the rectangular shortest-augmenting-path solver of Crouse 2016 that scipy implements) on
// rows 0..V-1 of cost_ce + cost_siou, by ONE warp: fp64 duals like scipy, the same evaluation order of every sum, and the same
// choice among equal path costs (scipy scans the remaining columns in order and lets a later column replace an equal earlier one
// only if it is unassigned: the winner is the LAST unassigned column among the minima if there is one, else the FIRST minimum --
// encoded below as a unique integer score per scan position, so the lane-parallel scan picks exactly scipy's column; checked
// against scipy on tie-heavy matrices in tests/test_gpu_train.py).  Then the matched loss terms (evaluator.py:27-36):
// loss3 = { mean cost_ce[g, col(g)], mean pred[:, unmatched columns] (0 if none), mean cost_siou[g, col(g)] }.
__global__ void __launch_bounds__(32) hungarian_assign_kernel(const float* __restrict__ cost_ce, const float* __restrict__ cost_siou,
                                                              const float* __restrict__ s_sum, const int32_t* __restrict__ n_valid_dev,
                                                              int64_t n, int k, int32_t* __restrict__ row_of_col,
                                                              float* __restrict__ loss3) {
  __shared__ double u[EV_MAX_K], v[EV_MAX_K], sp[EV_MAX_K];
  __shared__ int path[EV_MAX_K], col4row[EV_MAX_K], row4col[EV_MAX_K], remaining[EV_MAX_K];
  __shared__ unsigned char SR[EV_MAX_K], SC[EV_MAX_K];
  const int lane = threadIdx.x;
  const int V = *n_valid_dev;
  const float qnan = __int_as_float(0x7fc00000);
  if (V < 1 || V > k) {                                       // label_rows_kernel rejected the labels
    for (int p = lane; p < k; p += 32) row_of_col[p] = -1;
    if (lane < 3) loss3[lane] = qnan;
    return;
  }
  for (int j = lane; j < k; j += 32) { v[j] = 0.0; path[j] = -1; row4col[j] = -1; }
  for (int i = lane; i < V; i += 32) { u[i] = 0.0; col4row[i] = -1; }
  __syncwarp();
  const double INF = __longlong_as_double(0x7ff0000000000000LL);
  bool failed = false;
  for (int cur = 0; cur < V && !failed; ++cur) {
    for (int j = lane; j < k; j += 32) { remaining[j] = k - j - 1; SC[j] = 0; sp[j] = INF; }
    for (int i = lane; i < V; i += 32) SR[i] = 0;
    __syncwarp();
    double min_val = 0.0;
    int i = cur, sink = -1, R = k;
    while (sink < 0) {
      if (lane == 0) SR[i] = 1;
      const double ui = u[i];
      double best = INF;
      int bscore = -1, bit = -1;
      for (int it = lane; it < R; it += 32) {
        const int j = remaining[it];
        const double c = (double)__fadd_rn(__ldg(cost_ce + i * k + j), __ldg(cost_siou + i * k + j));      // evaluator.py:70 (fp32 sum)
        const double r = ((min_val + c) - ui) - v[j];
        double s = sp[j];
        if (r < s) { path[j] = i; sp[j] = r; s = r; }
        const int score = (row4col[j] < 0) ? R + it : R - 1 - it;
        if (s < best || (s == best && score > bscore)) { best = s; bscore = score; bit = it; }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        const double ob = __shfl_xor_sync(FULL, best, d);
        const int os = __shfl_xor_sync(FULL, bscore, d), oi = __shfl_xor_sync(FULL, bit, d);
        if (ob < best || (ob == best && os > bscore)) { best = ob; bscore = os; bit = oi; }
      }
      if (bit < 0 || !(best < INF)) { failed = true; break; }       // NaN / infinite costs: no finite augmenting path
      min_val = best;
      const int j = remaining[bit];
      const int r4c = row4col[j];
      if (r4c < 0) sink = j; else i = r4c;
      __syncwarp();
      if (lane == 0) { SC[j] = 1; remaining[bit] = remaining[R - 1]; }
      --R;
      __syncwarp();
    }
    if (failed) break;
    if (lane == 0) u[cur] += min_val;
    for (int i2 = lane; i2 < V; i2 += 32)
      if (SR[i2] && i2 != cur) u[i2] += min_val - sp[col4row[i2]];
    for (int j = lane; j < k; j += 32)
      if (SC[j]) v[j] -= min_val - sp[j];
    __syncwarp();
    if (lane == 0) {                                                // augment along the path
      int j = sink;
      while (true) {
        const int i2 = path[j];
        row4col[j] = i2;
        const int t = col4row[i2];
        col4row[i2] = j;
        j = t;
        if (i2 == cur) break;
      }
    }
    __syncwarp();
  }
  if (failed) {
    for (int p = lane; p < k; p += 32) row_of_col[p] = -1;
    if (lane < 3) loss3[lane] = qnan;
    return;
  }
  double ce = 0.0, si = 0.0, inv = 0.0;
  for (int g = lane; g < V; g += 32) { ce += (double)cost_ce[g * k + col4row[g]]; si += (double)cost_siou[g * k + col4row[g]]; }
  for (int p = lane; p < k; p += 32) {
    row_of_col[p] = row4col[p];
    if (row4col[p] < 0) inv += (double)s_sum[p];
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    ce += __shfl_xor_sync(FULL, ce, d); si += __shfl_xor_sync(FULL, si, d); inv += __shfl_xor_sync(FULL, inv, d);
  }
  if (lane == 0) {
    loss3[0] = (float)(ce / (double)V);
    loss3[1] = (k > V) ? (float)(inv / ((double)n * (double)(k - V))) : 0.0f;
    loss3[2] = (float)(si / (double)V);
  }
}

int launch_hungarian_costs(const float* pred, const int32_t* gt_row, int64_t n, int k, float* cost_ce, float* cost_siou,
                           float* tp, float* s_sum, float* cnt, cudaStream_t st) {
  DMN_CHECK(k >= 1 && k <= EV_MAX_K, "hungarian_costs: ins_num %d out of range (max %d)", k, EV_MAX_K);
  DMN_CHECK(n >= 1, "hungarian_costs: empty batch");
  hungarian_partials_kernel<true><<<(unsigned)k, HP_WARPS * 32, 0, st>>>(pred, gt_row, n, k, nullptr, cost_ce, cost_siou, tp, s_sum,
                                                                         cnt);
  DMN_LAUNCH_OK();
  return 0;
}

int launch_ins_loss_grad(const float* pred, const int32_t* gt_row, int64_t n, int64_t n_norm, int k, const int32_t* row_of_col,
                         const int32_t* n_valid, const float* tp, const float* s_sum, const float* cnt, const float* g3, float* d_pred,
                         cudaStream_t st) {
  DMN_CHECK(k >= 1 && k <= EV_MAX_K, "ins_loss_grad: ins_num %d out of range (max %d)", k, EV_MAX_K);
  DMN_CHECK(n_norm >= n, "ins_loss_grad: %lld rows of a batch of %lld", (long long)n, (long long)n_norm);
  const int64_t total = n * k;
  if (total == 0) return 0;
  ins_loss_grad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(pred, gt_row, n, n_norm, k, row_of_col, n_valid, tp, s_sum,
                                                                        cnt, g3, d_pred);
  DMN_LAUNCH_OK();
  return 0;
}

int launch_hungarian_partials(const float* pred, const int32_t* gt_row, int64_t n, int k, double* partials, cudaStream_t st) {
  DMN_CHECK(k >= 1 && k <= EV_MAX_K, "hungarian_partials: ins_num %d out of range (max %d)", k, EV_MAX_K);
  DMN_CHECK(n >= 0, "hungarian_partials: negative ray count");
  hungarian_partials_kernel<false><<<(unsigned)k, HP_WARPS * 32, 0, st>>>(pred, gt_row, n, k, partials, nullptr, nullptr, nullptr,
                                                                          nullptr, nullptr);
  DMN_LAUNCH_OK();
  return 0;
}

int launch_hungarian_costs_merged(const double* partials, int world, int64_t n, int k, float* cost_ce, float* cost_siou, float* tp,
                                  float* s_sum, float* cnt, cudaStream_t st) {
  DMN_CHECK(k >= 1 && k <= EV_MAX_K, "hungarian_costs_merged: ins_num %d out of range (max %d)", k, EV_MAX_K);
  DMN_CHECK(world >= 1 && n >= 1, "hungarian_costs_merged: %d shards of a batch of %lld rays", world, (long long)n);
  hungarian_costs_merged_kernel<<<(unsigned)k, 128, 0, st>>>(partials, world, n, k, cost_ce, cost_siou, tp, s_sum, cnt);
  DMN_LAUNCH_OK();
  return 0;
}

// Error word of the device-side assignment in mapped host memory (one per process): written by label_rows_kernel, read and
// cleared by ins_status_take() on the host without any synchronisation.
static volatile int32_t* g_ins_h_status = nullptr;
static int32_t* g_ins_d_status = nullptr;
static int ins_status_init() {
  if (g_ins_h_status) return 0;
  int32_t* h = nullptr;
  DMN_CUDA(cudaHostAlloc((void**)&h, sizeof(int32_t), cudaHostAllocMapped | cudaHostAllocPortable));
  *h = 0;
  DMN_CUDA(cudaHostGetDevicePointer((void**)&g_ins_d_status, (void*)h, 0));
  g_ins_h_status = h;
  return 0;
}
int ins_status_take() {
  if (!g_ins_h_status) return 0;
  const int code = (int)*g_ins_h_status;
  if (code) *g_ins_h_status = 0;
  return code;
}

int launch_label_rows(const int32_t* labels, int64_t n, int k, int32_t* gt_row, int32_t* n_valid, cudaStream_t st) {
  DMN_CHECK(k >= 1 && k <= EV_MAX_K, "ins_label_rows: ins_num %d out of range (max %d)", k, EV_MAX_K);
  DMN_CHECK(n >= 1, "ins_label_rows: empty batch");
  if (ins_status_init()) return 1;
  label_rows_kernel<<<1, 1024, 0, st>>>(labels, n, k, gt_row, n_valid, g_ins_d_status);
  DMN_LAUNCH_OK();
  return 0;
}

int launch_label_bitmap(const int32_t* labels, int64_t n, uint32_t* bitmap, cudaStream_t st) {
  DMN_CHECK(n >= 0, "ins_label_bitmap: negative ray count");
  if (ins_status_init()) return 1;
  label_bitmap_kernel<<<1, 1024, 0, st>>>(labels, n, bitmap, g_ins_d_status);
  DMN_LAUNCH_OK();
  return 0;
}

int launch_label_rows_merged(const uint32_t* bitmaps, int world, const int32_t* labels, int64_t n, int k, int32_t* gt_row,
                             int32_t* n_valid, cudaStream_t st) {
  DMN_CHECK(k >= 1 && k <= EV_MAX_K, "ins_label_rows_merged: ins_num %d out of range (max %d)", k, EV_MAX_K);
  DMN_CHECK(world >= 1 && n >= 0, "ins_label_rows_merged: %d shards, %lld rows", world, (long long)n);
  if (ins_status_init()) return 1;
  label_rows_merged_kernel<<<1, 1024, 0, st>>>(bitmaps, world, labels, n, k, gt_row, n_valid, g_ins_d_status);
  DMN_LAUNCH_OK();
  return 0;
}

int launch_hungarian_assign(const float* cost_ce, const float* cost_siou, const float* s_sum, const int32_t* n_valid, int64_t n, int k,
                            int32_t* row_of_col, float* loss3, cudaStream_t st) {
  DMN_CHECK(k >= 1 && k <= EV_MAX_K, "hungarian_assign: ins_num %d out of range (max %d)", k, EV_MAX_K);
  DMN_CHECK(n >= 1, "hungarian_assign: empty batch");
  hungarian_assign_kernel<<<1, 32, 0, st>>>(cost_ce, cost_siou, s_sum, n_valid, n, k, row_of_col, loss3);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
