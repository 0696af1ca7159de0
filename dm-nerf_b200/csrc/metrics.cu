// Test-view evaluation of render_test (networks/tester.py:87-128): PSNR and SSIM of the rendered image as scikit-image 0.18.3
// computes them, and the instance AP of ins_eval + calculate_ap (networks/evaluator.py:77-175, integral method).
//
// Every reduction that reaches a result runs in a fixed order (per-thread sums, block trees, one final block); the only atomics
// are integer counts.  Rules and deviations: DESIGN.md, "Evaluation metrics".
//
// Instance AP.  gt and prediction are both one-hot in ins_eval, so the reference's [K, K, N] broadcast is a joint histogram of
// the two label maps:  hist[g][l] = #{pixels with gt rank g and predicted label l}, built in one pass over the [N, K] instance
// map.  From it: cost_ce[g][c] = fl32(-log(1e-8)) * mismatches / N, cost_siou[g][c] = 1 - TP / (TP + FP + FN + 1e-6) (fp32 on
// exact integer counts, as the reference forms it), the assignment by the device LSAP solver of evaluator.cu, and the AP by one
// warp.  Per-label median confidences come from a radix sort of (label << 32 | ordered bits of the confidence).
#include <cub/device/device_radix_sort.cuh>

#include <cmath>
#include <cstdint>

#include "common.cuh"

namespace dmnerf {

namespace {

constexpr int MT = 256;                       // threads of the streaming kernels
constexpr int MAX_PARTS = 1024;               // partial sums of the PSNR pass
constexpr int SS_TW = 32, SS_TH = 16;         // SSIM output tile
constexpr int MK = DMNERF_MAX_INS + 1;        // labels 0..ins_num (ins_num = masked pixels)
constexpr int N_THRE = 6;
__constant__ float c_thre[N_THRE] = {0.5f, 0.75f, 0.8f, 0.85f, 0.9f, 0.95f};      // evaluator.py:10, compared in fp32

// Deterministic block sum (fixed tree) of one double per thread; every thread gets the total.
__device__ double block_sum(double v, double* sh) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < nw; ++w) s += sh[w];
  return s;
}

// ---------------------------------------------------------------------------------------------------------------- PSNR, SSIM
// mean_squared_error of skimage 0.18.3: difference and square in the input dtype (float32), mean in float64.
__global__ void __launch_bounds__(MT) psnr_parts_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n,
                                                        double* __restrict__ parts) {
  __shared__ double sh[32];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * MT + threadIdx.x; i < n; i += (int64_t)gridDim.x * MT) {
    const float d = __fsub_rn(a[i], b[i]);
    s += (double)__fmul_rn(d, d);
  }
  s = block_sum(s, sh);
  if (threadIdx.x == 0) parts[blockIdx.x] = s;
}

// structural_similarity(multichannel=True, data_range=1) of skimage 0.18.3 on one output tile of one channel: 7x7 uniform
// filter in float64 (each row window summed directly and divided by 7, then each column window of those), sample covariance
// (49/48), S averaged over the interior cropped by 3 pixels.  This equals scipy's uniform_filter (axis 0 first, running sums) to
// fp64 rounding, not bit for bit.  Only interior pixels are ever averaged, and their windows lie inside the image, so the
// filter's boundary mode never enters the result.
__global__ void __launch_bounds__(MT) ssim_tile_kernel(const float* __restrict__ x, const float* __restrict__ y, int H, int W,
                                                       double* __restrict__ parts) {
  __shared__ double hs[5][SS_TH + 6][SS_TW];
  __shared__ double sh[32];
  const int ch = blockIdx.z;
  const int r0 = 3 + blockIdx.y * SS_TH, c0 = 3 + blockIdx.x * SS_TW;       // first interior output of the tile
  for (int e = threadIdx.x; e < (SS_TH + 6) * SS_TW; e += MT) {
    const int rr = e / SS_TW, cc = e % SS_TW;
    const int r = r0 - 3 + rr, c = c0 + cc;
    double sx = 0.0, sy = 0.0, sxx = 0.0, syy = 0.0, sxy = 0.0;
    if (r < H && c < W - 3) {
      for (int k = -3; k <= 3; ++k) {
        const size_t o = ((size_t)r * W + (c + k)) * 3 + ch;
        const double u = (double)x[o], v = (double)y[o];
        sx += u; sy += v; sxx += u * u; syy += v * v; sxy += u * v;
      }
    }
    hs[0][rr][cc] = sx / 7.0; hs[1][rr][cc] = sy / 7.0; hs[2][rr][cc] = sxx / 7.0; hs[3][rr][cc] = syy / 7.0;
    hs[4][rr][cc] = sxy / 7.0;
  }
  __syncthreads();
  const double cov_norm = 49.0 / 48.0, C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
  double acc = 0.0;
  for (int e = threadIdx.x; e < SS_TH * SS_TW; e += MT) {
    const int rr = e / SS_TW, cc = e % SS_TW;
    const int r = r0 + rr, c = c0 + cc;
    if (r >= H - 3 || c >= W - 3) continue;
    double m[5];
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      double s = 0.0;
      for (int k = 0; k < 7; ++k) s += hs[q][rr + k][cc];
      m[q] = s / 7.0;
    }
    const double ux = m[0], uy = m[1];
    const double vx = cov_norm * (m[2] - ux * ux), vy = cov_norm * (m[3] - uy * uy), vxy = cov_norm * (m[4] - ux * uy);
    const double A1 = 2.0 * ux * uy + C1, A2 = 2.0 * vxy + C2, B1 = ux * ux + uy * uy + C1, B2 = vx + vy + C2;
    acc += (A1 * A2) / (B1 * B2);
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) parts[((size_t)ch * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = acc;
}

__global__ void __launch_bounds__(MT) image_finish_kernel(const double* __restrict__ psnr_parts, int n_psnr, int64_t n,
                                                          const double* __restrict__ ssim_parts, int n_ssim, int64_t interior,
                                                          dmnerf_eval_result* res) {
  __shared__ double sh[32];
  double s = 0.0;
  for (int i = threadIdx.x; i < n_psnr; i += MT) s += psnr_parts[i];
  const double sse = block_sum(s, sh);
  double m[3];
  for (int ch = 0; ch < 3; ++ch) {
    double t = 0.0;
    for (int i = threadIdx.x; i < n_ssim; i += MT) t += ssim_parts[(size_t)ch * n_ssim + i];
    m[ch] = block_sum(t, sh) / (double)interior;
  }
  if (threadIdx.x == 0) {
    const double mse = sse / (double)n;
    res->psnr = 10.0 * log10(1.0 / mse);                 // zero error: +inf, like numpy
    res->ssim = ((m[0] + m[1]) + m[2]) / 3.0;
  }
}

// ---------------------------------------------------------------------------------------------------------------- instance AP
// Ordered bits of a float: unsigned order = float order (NaN is rejected before).
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct InsWs {                                  // device workspace of dmnerf_ins_eval, carved from the caller's buffer
  int32_t* hist;        // [(gt_num + 1) x (k + 1)]: row gt_num = pixels without a gt rank, column k = masked pixels
  int32_t* status;      // [1]: 1 = NaN in the instance map
  int32_t* valid;       // [k]: predicted label of column c (torch.unique order, after the mask rule)
  int32_t* n_pred;      // [1]
  int32_t* gt_num_dev;  // [1]: rows of the assignment
  float* median;        // [k]: median confidence of column c
  float* cost_ce;       // [gt_num x k]
  float* cost_siou;     // [gt_num x k]
  float* col_sum;       // [k] zeros (the solver's loss terms are not used)
  int32_t* row_of_col;  // [k]
  float* loss3;         // [3]
  uint64_t* keys_in;    // [n]
  uint64_t* keys_out;   // [n]
  void* sort_tmp;
  size_t sort_bytes;
};

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

size_t sort_temp_bytes(int64_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n, 0, 40);
  return bytes;
}

size_t ins_ws_layout(int64_t n, int k, char* base, InsWs* w) {
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align_up(bytes); return (void*)p; };
  InsWs l;
  l.hist = (int32_t*)take((size_t)MK * (MK + 1) * 4);
  l.status = (int32_t*)take(4);
  l.valid = (int32_t*)take((size_t)MK * 4);
  l.n_pred = (int32_t*)take(4);
  l.gt_num_dev = (int32_t*)take(4);
  l.median = (float*)take((size_t)MK * 4);
  l.cost_ce = (float*)take((size_t)k * k * 4);
  l.cost_siou = (float*)take((size_t)k * k * 4);
  l.col_sum = (float*)take((size_t)k * 4);
  l.row_of_col = (int32_t*)take((size_t)k * 4);
  l.loss3 = (float*)take(16);
  l.keys_in = (uint64_t*)take((size_t)n * 8);
  l.keys_out = (uint64_t*)take((size_t)n * 8);
  l.sort_bytes = sort_temp_bytes(n);
  l.sort_tmp = take(l.sort_bytes);
  if (w) *w = l;
  return off;
}

// Per-pixel pass: predicted label = first maximum (torch.argmax), confidence = the maximum (np.max); masked pixels get label k
// (evaluator.py:127-132).  One privatised histogram per block in shared memory, flushed with integer atomics.
__global__ void __launch_bounds__(MT) ins_pixel_kernel(const float* __restrict__ ins, int64_t n, int k, const int32_t* __restrict__ gt_row,
                                                       int gt_num, const float* __restrict__ mask, const int32_t* __restrict__ mask_labels,
                                                       int mask_below, int64_t* __restrict__ pred_label, uint64_t* __restrict__ keys,
                                                       int32_t* __restrict__ hist, int32_t* __restrict__ status) {
  extern __shared__ int32_t sh_hist[];
  const int cols = k + 1, cells = (gt_num + 1) * cols;
  for (int e = threadIdx.x; e < cells; e += MT) sh_hist[e] = 0;
  __syncthreads();
  bool nan = false;
  for (int64_t i = (int64_t)blockIdx.x * MT + threadIdx.x; i < n; i += (int64_t)gridDim.x * MT) {
    const float* row = ins + i * k;
    float best = row[0];
    int arg = 0;
    nan |= best != best;
    for (int c = 1; c < k; ++c) {
      const float v = row[c];
      nan |= v != v;
      if (v > best) { best = v; arg = c; }
    }
    const bool masked = mask ? (mask[i] == 0.0f) : (mask_labels ? (mask_labels[i] >= mask_below) : false);
    const int lab = masked ? k : arg;
    const int g0 = gt_row[i];
    const int g = (g0 >= 0 && g0 < gt_num) ? g0 : gt_num;
    atomicAdd(&sh_hist[g * cols + lab], 1);
    pred_label[i] = lab;
    keys[i] = ((uint64_t)lab << 32) | f2key(best);
  }
  if (nan) atomicOr(status, 1);
  __syncthreads();
  for (int e = threadIdx.x; e < cells; e += MT)
    if (sh_hist[e]) atomicAdd(&hist[e], sh_hist[e]);
}

// Valid predicted labels, per-label median confidence and the two cost matrices, by one block.
__global__ void __launch_bounds__(1024) ins_costs_kernel(InsWs w, int64_t n, int k, int gt_num, int masked) {
  __shared__ int32_t colcnt[MK + 1], start[MK + 1], rowcnt[MK], valid[MK];
  __shared__ int n_valid;
  const int t = threadIdx.x, cols = k + 1;
  for (int l = t; l <= k; l += blockDim.x) {
    int s = 0;
    for (int g = 0; g <= gt_num; ++g) s += w.hist[g * cols + l];
    colcnt[l] = s;
  }
  for (int g = t; g < gt_num; g += blockDim.x) {
    int s = 0;
    for (int l = 0; l <= k; ++l) s += w.hist[g * cols + l];
    rowcnt[g] = s;
  }
  __syncthreads();
  if (t == 0) {
    // torch.unique(pred_label) ascending; with a mask the largest label present is dropped ([:-1], evaluator.py:133) -- label k
    // when a pixel is masked, otherwise the largest real label
    int s = 0, nv = 0, last = -1;
    for (int l = 0; l <= k; ++l) {
      start[l] = s;
      s += colcnt[l];
      if (colcnt[l] > 0) { last = l; if (l < k) valid[nv++] = l; }
    }
    if (masked && last >= 0 && last < k) --nv;
    n_valid = nv;
    *w.n_pred = nv;
    *w.gt_num_dev = gt_num;
  }
  __syncthreads();
  const int nv = n_valid;
  for (int c = t; c < k; c += blockDim.x) {
    float med = 0.0f;
    int lab = -1;
    if (c < nv) {
      lab = valid[c];
      const int cnt = colcnt[lab];
      const int64_t mid = (int64_t)start[lab] + cnt / 2;
      const float hi = key2f((uint32_t)w.keys_out[mid]);
      // np.median of float32: the middle element, or the float32 mean of the two middle ones
      med = (cnt & 1) ? hi : __fmul_rn(__fadd_rn(key2f((uint32_t)w.keys_out[mid - 1]), hi), 0.5f);
    }
    w.valid[c] = lab;
    w.median[c] = med;
    w.col_sum[c] = 0.0f;
  }
  const float ce = (float)(-log((double)1e-8f));             // -log(0 + 1e-8) = -log(1 - 1 + 1e-8) in fp32
  for (int e = t; e < gt_num * k; e += blockDim.x) {
    const int g = e / k, c = e % k;
    const int tp = c < nv ? w.hist[g * cols + valid[c]] : 0;
    const int cp = c < nv ? colcnt[valid[c]] : 0;
    const int cg = rowcnt[g];
    w.cost_ce[e] = (float)((double)ce * (double)(cg + cp - 2 * tp) / (double)n);
    const float tpf = (float)tp, fp = __fsub_rn((float)cp, tpf), fn = __fsub_rn((float)cg, tpf);
    const float den = __fadd_rn(__fadd_rn(__fadd_rn(tpf, fp), fn), 1e-6f);
    w.cost_siou[e] = __fsub_rn(1.0f, __fdiv_rn(tpf, den));
  }
}

// calculate_ap (evaluator.py:77-122, integral method) by one warp: lane t < 6 evaluates threshold t.  Matches are ordered by
// confidence, descending, ties in index order (stable); without confidences by IoU, descending.  Precision, recall and the
// integral's terms are the original's fp32 values; the terms are summed sequentially (torch.sum uses a vectorised cascade), so
// the AP equals the original's to fp32 rounding.
__device__ void warp_ap(const float* iou, const float* conf, int m, int gt_number, int* order, float* ap6) {
  const int lane = threadIdx.x & 31;
  if (lane == 0) {
    for (int i = 0; i < m; ++i) order[i] = i;
    for (int i = 1; i < m; ++i) {                              // stable insertion sort, m <= 128
      const int o = order[i];
      const float key = conf ? conf[o] : iou[o];
      int j = i - 1;
      while (j >= 0 && (conf ? conf[order[j]] : iou[order[j]]) < key) { order[j + 1] = order[j]; --j; }
      order[j + 1] = o;
    }
  }
  __syncwarp();
  if (lane < N_THRE) {
    const float thre = c_thre[lane];
    float mprec[MK + 2], mrec[MK + 2];
    mrec[0] = 0.0f; mprec[0] = 0.0f;
    int tp = 0;
    for (int i = 0; i < m; ++i) {
      tp += iou[order[i]] > thre ? 1 : 0;
      mprec[i + 1] = __fdiv_rn((float)tp, (float)(i + 1));               // cumsum / arange(1..m)
      mrec[i + 1] = __fdiv_rn((float)tp, (float)gt_number);              // cumsum.float() / gt_number
    }
    mrec[m + 1] = 1.0f; mprec[m + 1] = 0.0f;
    for (int i = m + 1; i > 0; --i) mprec[i - 1] = fmaxf(mprec[i - 1], mprec[i]);
    float ap = 0.0f;
    for (int i = 0; i <= m; ++i)
      if (mrec[i + 1] != mrec[i]) ap = __fadd_rn(ap, __fmul_rn(__fsub_rn(mrec[i + 1], mrec[i]), mprec[i + 1]));
    ap6[lane] = ap;
  }
  __syncwarp();
}

// The matched pairs of the assignment -> IoUs, confidences, APs and the matched predicted labels (evaluator.py:156-175).
__global__ void __launch_bounds__(32) ins_ap_kernel(InsWs w, int k, int gt_num, dmnerf_eval_result* res) {
  __shared__ int col_of_row[MK], order[MK];
  __shared__ float iou[MK], conf[MK], ap6[N_THRE];
  const int lane = threadIdx.x;
  for (int g = lane; g < gt_num; g += 32) col_of_row[g] = -1;
  __syncwarp();
  for (int c = lane; c < k; c += 32) {
    const int g = w.row_of_col[c];
    if (g >= 0 && g < gt_num) col_of_row[g] = c;
  }
  __syncwarp();
  const int nv = *w.n_pred;
  for (int g = lane; g < gt_num; g += 32) {
    const int c = col_of_row[g];
    iou[g] = c >= 0 ? __fsub_rn(1.0f, w.cost_siou[g * k + c]) : 0.0f;
    conf[g] = (c >= 0 && c < nv) ? w.median[c] : 0.0f;
    res->return_labels[g] = (c >= 0 && c < nv) ? w.valid[c] : -1;
  }
  __syncwarp();
  if (gt_num > 0) {
    warp_ap(iou, conf, gt_num, gt_num, order, ap6);
  } else if (lane < N_THRE) {
    ap6[lane] = 1.0f;                                              // no gt object in the frame
  }
  __syncwarp();
  if (lane < N_THRE) res->ap[lane] = ap6[lane];
  if (lane == 0) {
    res->gt_num = gt_num;
    res->pred_num = nv;
    bool matched = true;
    for (int g = 0; g < gt_num; ++g) matched &= col_of_row[g] >= 0;
    res->status = *w.status ? 1 : (matched ? 0 : 2);
  }
}

__global__ void __launch_bounds__(32) calculate_ap_kernel(const float* __restrict__ iou_in, const float* __restrict__ conf_in, int m,
                                                          int gt_number, float* __restrict__ ap_out) {
  __shared__ float iou[MK], conf[MK], ap6[N_THRE];
  __shared__ int order[MK];
  for (int i = threadIdx.x; i < m; i += 32) { iou[i] = iou_in[i]; conf[i] = conf_in ? conf_in[i] : 0.0f; }
  __syncwarp();
  warp_ap(iou, conf_in ? conf : nullptr, m, gt_number, order, ap6);
  if (threadIdx.x < N_THRE) ap_out[threadIdx.x] = ap6[threadIdx.x];
}

// gt_ins [n, k] one-hot (columns >= gt_num ignored) -> rank of the first set column, -1 if none.
__global__ void dense_rows_kernel(const float* __restrict__ gt, int64_t n, int k, int gt_num, int32_t* __restrict__ rows) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int r = -1;
  for (int c = 0; c < gt_num && r < 0; ++c)
    if (gt[i * k + c] != 0.0f) r = c;
  rows[i] = r;
}

template <typename T>
__global__ void label_colors_kernel(const T* __restrict__ labels, int64_t n, const uint8_t* __restrict__ lut, int n_lut,
                                    uint8_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t l = (int64_t)labels[i];
  uint8_t r = 0, g = 0, b = 0;
  if (l >= 0 && l < n_lut) { r = lut[3 * l]; g = lut[3 * l + 1]; b = lut[3 * l + 2]; }
  out[3 * i] = r; out[3 * i + 1] = g; out[3 * i + 2] = b;
}

int psnr_blocks(int64_t n3) { const int64_t b = (n3 + MT - 1) / MT; return (int)(b < MAX_PARTS ? b : MAX_PARTS); }

}  // namespace

int64_t eval_workspace_bytes(int64_t n, int k, int H, int W) {
  const size_t img = align_up((size_t)MAX_PARTS * 8) +
                     align_up((size_t)3 * ((W + SS_TW - 1) / SS_TW + 1) * ((H + SS_TH - 1) / SS_TH + 1) * 8);
  const size_t ins = (n > 0 && k > 0) ? ins_ws_layout(n, k, nullptr, nullptr) : 0;
  return (int64_t)(img > ins ? img : ins);
}

int eval_image(const float* rgb, const float* gt, int H, int W, void* ws, dmnerf_eval_result* res, cudaStream_t st) {
  DMN_CHECK(H >= 7 && W >= 7, "eval_image: %dx%d frame is smaller than the 7x7 SSIM window", H, W);
  const int64_t n3 = (int64_t)H * W * 3;
  const int pb = psnr_blocks(n3);
  double* psnr_parts = (double*)ws;
  double* ssim_parts = (double*)((char*)ws + align_up((size_t)MAX_PARTS * 8));
  psnr_parts_kernel<<<pb, MT, 0, st>>>(rgb, gt, n3, psnr_parts);
  DMN_LAUNCH_OK();
  const dim3 grid((W - 6 + SS_TW - 1) / SS_TW, (H - 6 + SS_TH - 1) / SS_TH, 3);
  ssim_tile_kernel<<<grid, MT, 0, st>>>(rgb, gt, H, W, ssim_parts);
  DMN_LAUNCH_OK();
  image_finish_kernel<<<1, MT, 0, st>>>(psnr_parts, pb, n3, ssim_parts, (int)(grid.x * grid.y), (int64_t)(H - 6) * (W - 6), res);
  DMN_LAUNCH_OK();
  return 0;
}

int ins_eval(const float* ins, int64_t n, int k, const int32_t* gt_row, int gt_num, const float* mask, const int32_t* mask_labels,
             int mask_below, int64_t* pred_label, void* ws, dmnerf_eval_result* res, cudaStream_t st) {
  DMN_CHECK(k >= 1 && k <= DMNERF_MAX_INS, "ins_eval: ins_num %d out of range [1, %d]", k, DMNERF_MAX_INS);
  DMN_CHECK(gt_num >= 0 && gt_num <= k, "ins_eval: %d gt objects for ins_num %d", gt_num, k);
  DMN_CHECK(n >= 1 && n < ((int64_t)1 << 31), "ins_eval: %lld pixels out of range", (long long)n);
  InsWs w;
  ins_ws_layout(n, k, (char*)ws, &w);
  const int cells = (gt_num + 1) * (k + 1);
  DMN_CUDA(cudaMemsetAsync(w.hist, 0, (size_t)cells * 4, st));
  DMN_CUDA(cudaMemsetAsync(w.status, 0, 4, st));
  static PerDeviceOnce once;
  if (once.first())
    DMN_CUDA(cudaFuncSetAttribute(ins_pixel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MK * (MK + 1) * 4));
  const int64_t nb64 = (n + MT - 1) / MT;
  const int nb = (int)(nb64 < 1056 ? nb64 : 1056);
  ins_pixel_kernel<<<nb, MT, (size_t)cells * 4, st>>>(ins, n, k, gt_row, gt_num, mask, mask_labels, mask_below, pred_label,
                                                      w.keys_in, w.hist, w.status);
  DMN_LAUNCH_OK();
  const int end_bit = 32 + (32 - __builtin_clz((unsigned)k));
  size_t need = 0;
  DMN_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, w.keys_in, w.keys_out, (int)n, 0, end_bit, st));
  DMN_CHECK(need <= w.sort_bytes, "ins_eval: sort workspace too small (%zu < %zu)", w.sort_bytes, need);
  DMN_CUDA(cub::DeviceRadixSort::SortKeys(w.sort_tmp, need, w.keys_in, w.keys_out, (int)n, 0, end_bit, st));
  g_launches.fetch_add(1);
  ins_costs_kernel<<<1, 1024, 0, st>>>(w, n, k, gt_num, (mask || mask_labels) ? 1 : 0);
  DMN_LAUNCH_OK();
  if (gt_num > 0) {
    if (launch_hungarian_assign(w.cost_ce, w.cost_siou, w.col_sum, w.gt_num_dev, n, k, w.row_of_col, w.loss3, st)) return 1;
  } else {
    DMN_CUDA(cudaMemsetAsync(w.row_of_col, 0xff, (size_t)k * 4, st));
  }
  ins_ap_kernel<<<1, 32, 0, st>>>(w, k, gt_num, res);
  DMN_LAUNCH_OK();
  return 0;
}

int calculate_ap(const float* iou, const float* conf, int m, int gt_number, float* ap6, cudaStream_t st) {
  DMN_CHECK(m >= 1 && m <= MK && gt_number >= 1, "calculate_ap: %d matches (max %d), gt_number %d", m, MK, gt_number);
  calculate_ap_kernel<<<1, 32, 0, st>>>(iou, conf, m, gt_number, ap6);
  DMN_LAUNCH_OK();
  return 0;
}

int ins_dense_rows(const float* gt_ins, int64_t n, int k, int gt_num, int32_t* rows, cudaStream_t st) {
  DMN_CHECK(gt_num >= 0 && gt_num <= k, "ins_dense_rows: gt_num %d > ins_num %d", gt_num, k);
  if (n == 0) return 0;
  dense_rows_kernel<<<(unsigned)((n + MT - 1) / MT), MT, 0, st>>>(gt_ins, n, k, gt_num, rows);
  DMN_LAUNCH_OK();
  return 0;
}

int label_colors(const void* labels, int is64, int64_t n, const uint8_t* lut, int n_lut, uint8_t* out, cudaStream_t st) {
  if (n == 0) return 0;
  const unsigned nb = (unsigned)((n + MT - 1) / MT);
  if (is64) label_colors_kernel<int64_t><<<nb, MT, 0, st>>>((const int64_t*)labels, n, lut, n_lut, out);
  else label_colors_kernel<int32_t><<<nb, MT, 0, st>>>((const int32_t*)labels, n, lut, n_lut, out);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
